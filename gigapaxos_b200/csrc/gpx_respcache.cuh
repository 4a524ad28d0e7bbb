/*
 * gpx_respcache.cuh -- the response cache's key table on the device (gpx_response_cache_*).  A node answers a client's
 * retransmitted request from its cache instead of proposing it again: PaxosManager.handleIncomingPacket :1084 checks
 * every incoming REQUEST against the cache (ENABLE_RESPONSE_CACHING, PaxosConfig.java:918), retransmittedRequest
 * :332-349 answers a hit, executed :311-330 fills the cache at every replica, and entries expire REQUEST_TIMEOUT after
 * they are put (GCConcurrentHashMap).  The table holds keys only; a cell names the response by the host's `handle`.
 *
 * Table: n_buckets (a power of two) buckets of GPX_RC_CELLS cells, one bucket = 320 bytes = 10 sectors.  A key is
 * (gid, generation, req_id, client address); the generation is the gid's count of gpx_set_group_names namings, so an
 * entry stops matching once its group has been named again.  A key's bucket is rc_hash's low bits, and no key ever
 * leaves its bucket.  A cell is live while its handle is >= 0 and now_ms - put_ms < timeout_ms.
 *
 * Every kernel here is scalar -- one thread per key, per request or per bucket run, plain loads and stores -- so
 * tests/emu compiles this file for the host.  The stable sorts and the scan between the launches are gpx_wire_seq.h's
 * rc_put and rc_match, run with CUB on the device and with the standard library in the emulation.
 */
#pragma once
#include "gpx_wire_dev.cuh"

#define GPX_RC_CELLS 8u

struct RcCell {  /* 40 B */
  uint32_t gid, gen;
  int64_t req_id;
  uint32_t ip;    /* rc_ip of the client address; 0 when port is 0 */
  uint16_t port;  /* 0 = no client address */
  uint16_t pad;
  int32_t handle; /* < 0: empty */
  int32_t pad2;
  int64_t put_ms;
};
static_assert(sizeof(RcCell) == 40 && sizeof(RcCell) * GPX_RC_CELLS % 32 == 0, "a bucket is whole sectors");

struct RcTable {
  RcCell* cell;         /* [mask + 1][GPX_RC_CELLS] */
  uint32_t mask;
  uint32_t G;           /* max_groups */
  int64_t timeout_ms;   /* >= 0 */
  const uint32_t* gen;  /* [G] the generation of each gid; nullptr without name state (generation 0) */
  const uint32_t* slot; /* [G] WireNames.slot; nullptr without name state (every gid counts as named) */
};

/* ---- the key --------------------------------------------------------------------------------------------------- */
__host__ __device__ __forceinline__ uint64_t rc_splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
/* the client address as a big-endian word; an absent address (port 0) is 0 whatever its bytes */
__host__ __device__ __forceinline__ uint32_t rc_ip(const uint8_t* ip, uint16_t port) {
  if (port == 0) return 0;
  return ((uint32_t)ip[0] << 24) | ((uint32_t)ip[1] << 16) | ((uint32_t)ip[2] << 8) | (uint32_t)ip[3];
}
/* h = splitmix64(req_id ^ splitmix64(gid << 32 | gen) ^ splitmix64(ip << 16 | port)); the bucket is h & mask */
__host__ __device__ __forceinline__ uint64_t rc_hash(uint32_t gid, uint32_t gen, int64_t req_id, uint32_t ip,
                                                     uint16_t port) {
  return rc_splitmix64((uint64_t)req_id ^ rc_splitmix64(((uint64_t)gid << 32) | gen) ^
                       rc_splitmix64(((uint64_t)ip << 16) | port));
}
__device__ __forceinline__ uint32_t rc_gen(const RcTable& T, uint32_t gid) { return T.gen ? T.gen[gid] : 0u; }

/* live: taken and not expired (now_ms - put_ms < timeout_ms, exact over the whole int64 range) */
__device__ __forceinline__ bool rc_live(const RcCell& c, int64_t now_ms, int64_t timeout_ms) {
  if (c.handle < 0) return false;
  if (now_ms < c.put_ms) return true;
  return (uint64_t)now_ms - (uint64_t)c.put_ms < (uint64_t)timeout_ms;
}
__device__ __forceinline__ bool rc_same(const RcCell& c, uint32_t gid, uint32_t gen, int64_t req_id, uint32_t ip,
                                        uint16_t port) {
  return c.gid == gid && c.gen == gen && c.req_id == req_id && c.ip == ip && c.port == port;
}
/* the lowest live cell of bucket b that holds the key, or -1 */
__device__ __forceinline__ int rc_find(const RcTable& T, const RcCell* b, uint32_t gid, uint32_t gen, int64_t req_id,
                                       uint32_t ip, uint16_t port, int64_t now_ms) {
  for (int c = 0; c < (int)GPX_RC_CELLS; c++)
    if (rc_live(b[c], now_ms, T.timeout_ms) && rc_same(b[c], gid, gen, req_id, ip, port)) return c;
  return -1;
}

/* ---- names: a gid's generation rises by one each time gpx_set_group_names names it ------------------------------- */
__global__ void k_rc_gen_bump(uint32_t* gen, const __grid_constant__ NameSetArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < A.n) gen[A.gids[k]]++; /* the gids of one call are distinct */
}

/* ---- put: executed requests' keys into the table ------------------------------------------------------------------
 * k_rc_put_keys checks every key and gives it its bucket and generation; the host sorts the keys by bucket, stably,
 * and k_rc_put gives each bucket's run one thread that applies the run's keys in input order. */
struct RcPutArgs {
  const gpx_rc_key* keys;
  uint32_t n;
  int64_t now_ms;
  uint32_t* bucket;      /* [n] */
  uint32_t* gen;         /* [n] the generation of the key's gid at the call */
  uint32_t* bad;         /* [1] zeroed by the host: set when a key has a negative handle or gid >= G */
  const uint32_t* perm;  /* [n] key indices in bucket order (stable) */
  const uint32_t* sbucket; /* [n] the buckets in that order */
};

__global__ void k_rc_put_keys(const __grid_constant__ RcTable T, const __grid_constant__ RcPutArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const gpx_rc_key k = A.keys[i];
  uint32_t gen = 0, b = 0;
  if (k.handle < 0 || k.gid >= T.G) {
    *A.bad = 1;
  } else {
    gen = rc_gen(T, k.gid);
    b = (uint32_t)(rc_hash(k.gid, gen, k.req_id, rc_ip(k.client_ip, k.client_port), k.client_port) & T.mask);
  }
  A.bucket[i] = b;
  A.gen[i] = gen;
}

/* one key into bucket b: over a live cell with the same key, else into the lowest free or expired cell, else over the
 * cell with the smallest put time (the lowest such cell) */
__device__ __forceinline__ void rc_apply(const RcTable& T, RcCell* b, const gpx_rc_key& k, uint32_t gen,
                                         int64_t now_ms) {
  const uint32_t ip = rc_ip(k.client_ip, k.client_port);
  int to = rc_find(T, b, k.gid, gen, k.req_id, ip, k.client_port, now_ms);
  if (to < 0) {
    int oldest = 0;
    for (int c = 0; c < (int)GPX_RC_CELLS && to < 0; c++) {
      if (!rc_live(b[c], now_ms, T.timeout_ms)) to = c;
      else if (b[c].put_ms < b[oldest].put_ms) oldest = c;
    }
    if (to < 0) to = oldest;
  }
  RcCell c;
  c.gid = k.gid;
  c.gen = gen;
  c.req_id = k.req_id;
  c.ip = ip;
  c.port = k.client_port;
  c.pad = 0;
  c.handle = k.handle;
  c.pad2 = 0;
  c.put_ms = now_ms;
  b[to] = c;
}

__global__ void k_rc_put(const __grid_constant__ RcTable T, const __grid_constant__ RcPutArgs A) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.n || (j > 0 && A.sbucket[j - 1] == A.sbucket[j])) return;
  const uint32_t bk = A.sbucket[j];
  RcCell* b = T.cell + (size_t)bk * GPX_RC_CELLS;
  for (uint32_t r = j; r < A.n && A.sbucket[r] == bk; r++) {
    const uint32_t i = A.perm[r];
    rc_apply(T, b, A.keys[i], A.gen[i], A.now_ms);
  }
}

/* ---- match: which requests the cache answers ------------------------------------------------------------------------
 * The host sorts the requests' client values, stably; k_rc_dups marks every request whose client value another request
 * of the call shares (a request unrolled from a batched RequestPacket), k_rc_match looks the others up, and after an
 * exclusive scan of the misses k_rc_scatter copies them in input order. */
struct RcMatchArgs {
  const gpx_request_rec* reqs;
  const gpx_wire_req_meta* meta;
  uint32_t n;
  int64_t now_ms;
  const uint32_t* perm;    /* [n] request indices in client order (stable) */
  const uint32_t* sclient; /* [n] the client values in that order */
  uint32_t* dup;           /* [n] 1: another request has the same client value */
  int32_t* hit;            /* [n] the cell's handle, or -1 */
  uint32_t* miss;          /* [n] 1 for a miss */
  const uint32_t* off;     /* [n] exclusive prefix sums of miss */
  gpx_request_rec* out_reqs;
  gpx_wire_req_meta* out_meta;
};

__global__ void k_rc_dups(const __grid_constant__ RcMatchArgs A) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= A.n) return;
  const uint32_t c = A.sclient[j];
  A.dup[A.perm[j]] = (j > 0 && A.sclient[j - 1] == c) || (j + 1 < A.n && A.sclient[j + 1] == c);
}

__global__ void k_rc_match(const __grid_constant__ RcTable T, const __grid_constant__ RcMatchArgs A) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= A.n) return;
  int32_t h = -1;
  const uint32_t gid = A.reqs[q].gid;
  if (!A.dup[q] && gid < T.G && (T.slot == nullptr || T.slot[gid] != GPX_NAME_NONE)) {
    const gpx_wire_req_meta& m = A.meta[q];
    const uint32_t gen = rc_gen(T, gid), ip = rc_ip(m.client_ip, m.client_port);
    const int64_t req_id = A.reqs[q].req_id;
    const RcCell* b = T.cell + (size_t)(rc_hash(gid, gen, req_id, ip, m.client_port) & T.mask) * GPX_RC_CELLS;
    const int c = rc_find(T, b, gid, gen, req_id, ip, m.client_port, A.now_ms);
    if (c >= 0) h = b[c].handle;
  }
  A.hit[q] = h;
  A.miss[q] = h < 0;
}

__global__ void k_rc_scatter(const __grid_constant__ RcMatchArgs A) {
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= A.n || !A.miss[q]) return;
  A.out_reqs[A.off[q]] = A.reqs[q];
  A.out_meta[A.off[q]] = A.meta[q];
}
