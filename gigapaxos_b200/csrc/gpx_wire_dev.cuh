/*
 * gpx_wire_dev.cuh -- the phase-2 wire codec on the device: a batch of received AcceptPacket / BatchedAcceptReply /
 * BatchedCommit bytes becomes engine records, and the engine's reply and decision records become BATCHED_ACCEPT_REPLY
 * and BATCHED_COMMIT bytes, coalesced as one PaxosPacketBatcher per node does (PaxosPacketBatcher.java:97-179,
 * 345-454).  Byte layouts: include/gpx_wire.h; the host codec there (gpx_wire.cpp) is the reference these kernels are
 * tested against.
 *
 * Names: a packet names its group by (paxosID, version) (PaxosPacket.java:459-476).  gpx_set_group_names stores, per
 * gid, the paxosID bytes and the version, and an open-addressing table from the bytes to the gid, probed from the Java
 * String.hashCode of the name; a hit is confirmed by comparing the bytes.
 *
 * Every kernel here is scalar -- one thread per packet, per record or per coalesced run, plain loads and stores over
 * gpx_dev.cuh's state -- so tests/emu compiles this file for the host.  The scans that size the outputs and the stable
 * sorts by gid run between the launches, in the sequences of gpx_wire_seq.h (CUB on the device, the standard library
 * in the emulation).
 */
#pragma once
#include "gpx_dev.cuh"
#include "gpx_wire.h"

#define GPX_NAME_BYTES 128u           /* per gid: length byte + up to GPX_WIRE_MAX_ID bytes */
#define GPX_NAME_EMPTY 0u             /* table key: never used */
#define GPX_NAME_TOMB 0xffffffffu     /* table key: removed */
#define GPX_NAME_NONE 0xffffffffu     /* WireNames.slot: the gid has no name */
#define GPX_WIRE_NOKEY 0xffffffffu    /* sort key of a record that is not encoded */

struct WireNames {
  uint2* tab;       /* [mask + 1] {gid + 1 (GPX_NAME_EMPTY / GPX_NAME_TOMB), String.hashCode} */
  uint32_t mask;
  uint8_t* name;    /* [G][GPX_NAME_BYTES] */
  int32_t* version; /* [G] */
  uint32_t* slot;   /* [G] table index of the gid's entry, GPX_NAME_NONE if it has none */
};

/* ---- big-endian reads (java.nio.ByteBuffer) ---------------------------------------------------------------------- */
struct WireRd {
  const uint8_t* p;
  uint32_t len, n;
  bool ok;
};
__device__ __forceinline__ WireRd wr_open(const uint8_t* p, uint32_t len, bool ok) {
  WireRd r;
  r.p = p;
  r.len = len;
  r.n = 0;
  r.ok = ok;
  return r;
}
__device__ __forceinline__ bool wr_need(WireRd& r, uint32_t k) {
  if (!r.ok || k > r.len - r.n) {
    r.ok = false;
    return false;
  }
  return true;
}
__device__ __forceinline__ uint32_t wr_u8(WireRd& r) {
  if (!wr_need(r, 1)) return 0;
  return r.p[r.n++];
}
__device__ __forceinline__ int32_t wr_i32(WireRd& r) {
  if (!wr_need(r, 4)) return 0;
  const uint8_t* q = r.p + r.n;
  r.n += 4;
  return (int32_t)(((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | (uint32_t)q[3]);
}
__device__ __forceinline__ int64_t wr_i64(WireRd& r) {
  const uint32_t hi = (uint32_t)wr_i32(r), lo = (uint32_t)wr_i32(r);
  return (int64_t)(((uint64_t)hi << 32) | lo);
}
__device__ __forceinline__ void wr_skip(WireRd& r, uint32_t k) {
  if (wr_need(r, k)) r.n += k;
}
/* a length field followed by that many bytes; a negative length is malformed */
__device__ __forceinline__ uint32_t wr_bytes(WireRd& r, uint32_t* at) {
  const int32_t l = wr_i32(r);
  if (l < 0) r.ok = false;
  *at = r.n;
  wr_skip(r, (uint32_t)l);
  return r.ok ? (uint32_t)l : 0u;
}

/* PaxosPacket header :459-476 */
struct WireHdr {
  int32_t type, version;
  uint32_t id_at, id_len;
};
__device__ __forceinline__ bool wr_header(WireRd& r, WireHdr& h) {
  const int32_t pp = wr_i32(r);
  h.type = wr_i32(r);
  h.version = wr_i32(r);
  h.id_len = wr_u8(r);
  h.id_at = r.n;
  wr_skip(r, h.id_len);
  return r.ok && pp == GPX_PT_PAXOS_PACKET && h.id_len <= GPX_WIRE_MAX_ID;
}
#define GPX_PT_BIT(t) (1ull << (t))
/* packet ref of the arena bytes[0..n_bytes): its reader r and header h.  GPX_WS_UNHANDLED for a JSON packet or a type
 * outside `types` (GPX_PT_BIT of each), GPX_WS_MALFORMED for a span past the arena or a bad header, else GPX_WS_OK with
 * r just past the header */
__device__ __forceinline__ int32_t wr_packet(const uint8_t* bytes, uint64_t n_bytes, const gpx_wire_ref& ref,
                                             uint64_t types, WireRd& r, WireHdr& h) {
  r = wr_open(bytes + ref.off, ref.len, (uint64_t)ref.off + ref.len <= n_bytes);
  if (r.ok && ref.len > 0 && r.p[0] == '{') return GPX_WS_UNHANDLED; /* JSON packet */
  if (!wr_header(r, h)) return GPX_WS_MALFORMED;
  if ((uint32_t)h.type >= 64u || !(types & GPX_PT_BIT(h.type))) return GPX_WS_UNHANDLED;
  return GPX_WS_OK;
}

/* RequestPacket(ByteBuffer) :956-1024 up to the batched requests: the fields the engine keeps */
struct WireReq {
  int64_t req_id;
  uint32_t stop;
  int32_t entry;
  uint32_t val_at, val_len;
  int32_t n_batched;
};
/* the fields the engine does not keep, for the REQUEST decoder (gpx_wire_req_meta) */
struct WireReqMore {
  gpx_wire_req_meta m;
  uint32_t digest_len, resp_len;
};
__device__ __forceinline__ uint32_t wr_u16(WireRd& r) {
  const uint32_t hi = wr_u8(r);
  return (hi << 8) | wr_u8(r);
}
/* x == nullptr (k_wire_decode): the other fields are skipped */
__device__ __forceinline__ void wr_request_body(WireRd& r, WireReq& q, WireReqMore* x = nullptr) {
  q.req_id = wr_i64(r);
  q.stop = wr_u8(r) == 1u;
  if (x) {
    for (int b = 0; b < 4; b++) x->m.client_ip[b] = (uint8_t)wr_u8(r);
    x->m.client_port = (uint16_t)wr_u16(r);
    for (int b = 0; b < 4; b++) x->m.listen_ip[b] = (uint8_t)wr_u8(r);
    x->m.listen_port = (uint16_t)wr_u16(r);
  } else {
    wr_skip(r, 4 + 2 + 4 + 2); /* client and listen addresses */
  }
  q.entry = wr_i32(r);
  if (x) {
    x->m.entry_time = wr_i64(r);
    x->m.flags = wr_u8(r) == 1u ? GPX_RM_RETURN_VALUE : 0u;
    x->m.forward_count = wr_i32(r);
    x->m.flags |= wr_u8(r) == 1u ? GPX_RM_BROADCASTED : 0u;
    x->m.pad = 0;
  } else {
    wr_skip(r, 8 + 1 + 4 + 1); /* entryTime, shouldReturnRequestValue, forwardCount, broadcasted */
  }
  uint32_t at;
  const uint32_t dl = wr_bytes(r, &at); /* digest */
  q.val_len = wr_bytes(r, &q.val_at);
  const uint32_t rl = wr_bytes(r, &at); /* responseValue */
  if (x) {
    x->digest_len = dl;
    x->resp_len = rl;
  }
  q.n_batched = wr_i32(r);
  if (q.n_batched < 0) r.ok = false;
}

/* the next latched request {int length}{REQUEST packet} (:929-936) at r.n: its reader s and body sq.  False (r.ok
 * false) when it does not fit in r, or is not a whole REQUEST packet without latched requests of its own
 * (RequestBatcher latches one level). */
__device__ __forceinline__ bool wr_latched(WireRd& r, WireRd& s, WireReq& sq, WireReqMore* sx) {
  const int32_t l = wr_i32(r);
  if (l < 0 || !wr_need(r, (uint32_t)l)) {
    r.ok = false;
    return false;
  }
  s = wr_open(r.p + r.n, (uint32_t)l, true);
  WireHdr sh;
  const bool hok = wr_header(s, sh);
  wr_request_body(s, sq, sx);
  if (!hok || !s.ok || sq.n_batched != 0 || s.n != s.len) r.ok = false;
  r.n += (uint32_t)l;
  return r.ok;
}
/* a request body and its latched requests, as AcceptPacket and RequestPacket carry them */
struct WireBatch {
  uint32_t sub_at, n_sub; /* where the latched requests start in r, and how many there are */
  uint32_t val, pay;      /* all value bytes, and the same with each value padded to 16 */
  uint32_t stop;          /* one of the requests is a STOP */
  bool host_only;         /* with x: one carries a digest or a responseValue */
};
__device__ __forceinline__ void wr_request_batch(WireRd& r, WireReq& q, WireReqMore* x, WireBatch& B) {
  wr_request_body(r, q, x);
  B.sub_at = r.n;
  B.n_sub = r.ok ? (uint32_t)q.n_batched : 0u;
  B.val = q.val_len;
  B.pay = (q.val_len + 15u) & ~15u;
  B.stop = q.stop;
  B.host_only = x && (x->digest_len != 0 || x->resp_len != 0);
  for (uint32_t b = 0; b < B.n_sub && r.ok; b++) {
    WireRd s;
    WireReq sq;
    WireReqMore sx;
    if (!wr_latched(r, s, sq, x ? &sx : nullptr)) break;
    B.val += sq.val_len;
    B.pay += (sq.val_len + 15u) & ~15u;
    B.stop |= sq.stop;
    B.host_only = B.host_only || (x && (sx.digest_len != 0 || sx.resp_len != 0));
  }
}

__device__ __forceinline__ void wire_copy(uint8_t* d, const uint8_t* s, uint32_t n) {
  for (uint32_t i = 0; i < n; i++) d[i] = s[i];
}

__device__ __forceinline__ uint32_t wire_popc(uint32_t m) { /* scalar: the emulation has no __popc */
  uint32_t c = 0;
  for (; m; m &= m - 1) c++;
  return c;
}

/* ---- names ----------------------------------------------------------------------------------------------------- */
__device__ __forceinline__ int32_t wire_name_hash(const uint8_t* s, uint32_t n) { /* String.hashCode (ISO-8859-1) */
  uint32_t h = 0;
  for (uint32_t i = 0; i < n; i++) h = 31u * h + s[i];
  return (int32_t)h;
}
__device__ __forceinline__ bool wire_name_eq(const WireNames& W, uint32_t gid, const uint8_t* s, uint32_t n) {
  const uint8_t* m = W.name + (size_t)gid * GPX_NAME_BYTES;
  if (m[0] != n) return false;
  for (uint32_t i = 0; i < n; i++)
    if (m[1 + i] != s[i]) return false;
  return true;
}
/* gid named s[0..n), or GPX_NAME_NONE */
__device__ __forceinline__ uint32_t wire_name_find(const WireNames& W, const uint8_t* s, uint32_t n) {
  const uint32_t h = (uint32_t)wire_name_hash(s, n);
  uint32_t i = h & W.mask;
  for (uint32_t probe = 0; probe <= W.mask; probe++, i = (i + 1) & W.mask) {
    const uint2 e = W.tab[i];
    if (e.x == GPX_NAME_EMPTY) break;
    if (e.x != GPX_NAME_TOMB && e.y == h && wire_name_eq(W, e.x - 1u, s, n)) return e.x - 1u;
  }
  return GPX_NAME_NONE;
}

/* enters gid (its bytes already stored) at the first free or removed cell of its probe sequence */
__device__ __forceinline__ void wire_name_put(const WireNames& W, uint32_t gid, bool reuse_tomb) {
  const uint8_t* m = W.name + (size_t)gid * GPX_NAME_BYTES;
  const uint32_t h = (uint32_t)wire_name_hash(m + 1, m[0]);
  uint32_t i = h & W.mask;
  for (;;) {
    const uint32_t cur = W.tab[i].x;
    if (cur == GPX_NAME_EMPTY || (reuse_tomb && cur == GPX_NAME_TOMB)) {
      if (atomicCAS(&W.tab[i].x, cur, gid + 1u) == cur) {
        W.tab[i].y = h;
        W.slot[gid] = i;
        return;
      }
      continue; /* another insert took the cell: look at it again */
    }
    i = (i + 1) & W.mask;
  }
}

/* one name per thread: the gid's bytes and version are already stored (host copy); the caller guarantees that no live
 * gid has the same name and that the table has free cells */
struct NameSetArgs {
  const uint32_t* gids;
  uint32_t n;
};
__global__ void k_names_insert(const __grid_constant__ WireNames W, const __grid_constant__ NameSetArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < A.n) wire_name_put(W, A.gids[k], true);
}
/* removes the entries of the given gids (gids without one are skipped) */
__global__ void k_names_remove(const __grid_constant__ WireNames W, const __grid_constant__ NameSetArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= A.n) return;
  const uint32_t gid = A.gids[k];
  const uint32_t s = W.slot[gid];
  if (s == GPX_NAME_NONE) return;
  W.tab[s].x = GPX_NAME_TOMB;
  W.slot[gid] = GPX_NAME_NONE;
}
/* with the table cleared: re-enters every named gid (the removed cells become free again) */
__global__ void k_names_rehash(const __grid_constant__ WireNames W, uint32_t G) {
  const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;
  if (gid < G && W.slot[gid] != GPX_NAME_NONE) wire_name_put(W, gid, false);
}
/* a batch of names staged as [n][GPX_NAME_BYTES] (length byte + bytes): found[k] = the gid that has name k now, or
 * GPX_NAME_NONE (gpx_set_group_names refuses a name another live gid holds before it changes anything) */
__global__ void k_names_find(const __grid_constant__ WireNames W, const uint8_t* staged, uint32_t n, uint32_t* found) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint8_t* m = staged + (size_t)k * GPX_NAME_BYTES;
  found[k] = wire_name_find(W, m + 1, m[0]);
}
/* stores name k and version k of the batch at gids[k] */
__global__ void k_names_store(const __grid_constant__ WireNames W, const __grid_constant__ NameSetArgs A,
                              const uint8_t* staged, const int32_t* version) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= A.n) return;
  wire_copy(W.name + (size_t)A.gids[k] * GPX_NAME_BYTES, staged + (size_t)k * GPX_NAME_BYTES, GPX_NAME_BYTES);
  W.version[A.gids[k]] = version[k];
}

/* ---- decode ---------------------------------------------------------------------------------------------------- */
enum { WD_ACC = 0, WD_BLOB = 1, WD_REP = 2, WD_DEC = 3, WD_NCNT = 4 };

struct WireDecodeArgs {
  const uint8_t* bytes;
  const gpx_wire_ref* pkts;
  uint64_t n_bytes;
  uint32_t n;
  uint32_t* cnt;  /* [WD_NCNT][n]: pass 0 writes the packet's output sizes (blob bytes padded to 16) */
  uint32_t* off;  /* [WD_NCNT][n]: pass 1 reads their exclusive prefix sums */
  int32_t* status;
  /* pass 1: records staged in packet order, and the sort keys (gids) beside them; the blob is the output itself */
  gpx_accept_rec* acc;
  uint8_t* blob;
  gpx_accept_reply_rec* rep;
  gpx_decision_rec* dec;
  uint32_t* acc_key;
  uint32_t* rep_key;
  uint32_t* dec_key;
  int emit;
};

__device__ __forceinline__ uint8_t wire_member_idx(const MsetInfo* ms, uint32_t R, int32_t node) {
  for (uint32_t i = 0; i < R; i++)
    if (ms->nodes[i] == node) return (uint8_t)i;
  return 0xffu;
}
/* entry-lane bits of gpx_request_rec.flags: the lane serving the entry replica, 0xf when that node is not local */
__device__ __forceinline__ uint32_t wire_entry_bits(const DevState& S, int32_t entry) {
  for (uint32_t l = 0; l < S.L; l++)
    if (S.lane_node[l] == entry) return l << 8;
  return 0xfu << 8;
}
/* gid (wire_name_find's, GPX_NAME_NONE included) as a packet's group at the packet's version: GPX_WS_UNKNOWN_NAME
 * without a live gid, GPX_WS_VERSION at another version (PISM :441-447), else GPX_WS_OK with its context in g */
__device__ __forceinline__ int32_t wire_group(const DevState& S, const WireNames& W, uint32_t gid, int32_t version,
                                              GroupCtx& g) {
  g = group_ctx(S, gid);
  if (gid == GPX_NAME_NONE || !g.live) return GPX_WS_UNKNOWN_NAME;
  if (W.version[gid] != version) return GPX_WS_VERSION;
  return GPX_WS_OK;
}
/* a request's receiving node: the lane serving it, which must also be a member of g (else GPX_WS_NOT_LOCAL) */
__device__ __forceinline__ int32_t wire_recv_lane(const DevState& S, const GroupCtx& g, int32_t node, uint32_t& lane) {
  lane = S.L;
  for (uint32_t l = 0; l < S.L; l++)
    if (S.lane_node[l] == node) lane = l;
  return lane == S.L || wire_member_idx(g.ms, g.R, node) == 0xffu ? GPX_WS_NOT_LOCAL : GPX_WS_OK;
}
/* the records a BatchedAcceptReply / BatchedCommit gives per slot, but the slot (and a reply's requestID) */
__device__ __forceinline__ gpx_accept_reply_rec wire_reply_rec(uint32_t gid, int32_t bnum, int32_t bcoord,
                                                               int32_t max_cp, uint32_t who) {
  gpx_accept_reply_rec x;
  x.gid = gid;
  x.slot = 0;
  x.bnum = bnum;
  x.bcoord = bcoord;
  x.max_cp = max_cp;
  x.who = who;
  x.req_id = 0;
  return x;
}
__device__ __forceinline__ gpx_decision_rec wire_decision_rec(uint32_t gid, int32_t bnum, int32_t bcoord,
                                                              int32_t median, uint16_t dst_mask) {
  gpx_decision_rec d;
  d.gid = gid;
  d.slot = 0;
  d.bnum = bnum;
  d.bcoord = bcoord;
  d.median_cp = median;
  d.flags = GPX_F_DECISION;
  d.dst_mask = dst_mask;
  d.req_id = 0; /* a BatchedCommit carries slots only: the value is the accept the acceptor holds */
  return d;
}

/* one thread per packet.  Pass 0 (emit == 0) parses and validates the packet, looks its name up and writes its status
 * and output sizes; pass 1 parses it again and writes its records at the scanned offsets. */
__global__ void k_wire_decode(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                              const __grid_constant__ WireDecodeArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= A.n) return;
  if (A.emit && A.status[k] != GPX_WS_OK) return;
  const gpx_wire_ref ref = A.pkts[k];
  uint32_t c[WD_NCNT] = {0, 0, 0, 0};
  WireRd r;
  WireHdr h;
  int32_t st = wr_packet(A.bytes, A.n_bytes, ref,
                         GPX_PT_BIT(GPX_PT_ACCEPT) | GPX_PT_BIT(GPX_PT_BATCHED_ACCEPT_REPLY) |
                             GPX_PT_BIT(GPX_PT_BATCHED_COMMIT),
                         r, h);
  /* body: parsed in full before anything is looked up, so a malformed packet is malformed whatever its name */
  WireReq q;
  WireBatch B = {};
  int32_t slot = 0, bnum = 0, bcoord = 0, median = 0, sender = 0, acceptor = 0, max_cp = 0, cnt_slots = 0, n_group = 0;
  uint32_t slots_at = 0;
  if (st == GPX_WS_OK) {
    if (h.type == GPX_PT_ACCEPT) { /* AcceptPacket :95-138 */
      wr_request_batch(r, q, nullptr, B);
      slot = wr_i32(r);
      bnum = wr_i32(r);
      bcoord = wr_i32(r);
      wr_u8(r); /* recovery */
      median = wr_i32(r);
      wr_u8(r); /* noCoalesce */
      sender = wr_i32(r);
    } else if (h.type == GPX_PT_BATCHED_ACCEPT_REPLY) { /* BatchedAcceptReply :103-173 */
      acceptor = wr_i32(r);
      bnum = wr_i32(r);
      bcoord = wr_i32(r);
      wr_i32(r); /* slotNumber of the first reply: also in the map */
      max_cp = wr_i32(r);
      wr_skip(r, 8 + 1); /* requestID, undigestRequest */
      cnt_slots = wr_i32(r);
      if (cnt_slots < 0 || (r.ok && (uint64_t)cnt_slots * 12u > r.len - r.n)) r.ok = false;
      slots_at = r.n;
      if (r.ok) wr_skip(r, (uint32_t)cnt_slots * 12u);
    } else { /* BatchedCommit :184-252 */
      bnum = wr_i32(r);
      bcoord = wr_i32(r);
      median = wr_i32(r);
      cnt_slots = wr_i32(r);
      if (cnt_slots < 0 || (r.ok && (uint64_t)cnt_slots * 4u > r.len - r.n)) r.ok = false;
      slots_at = r.n;
      if (r.ok) wr_skip(r, (uint32_t)cnt_slots * 4u);
      n_group = wr_i32(r);
      if (n_group < 0 || (r.ok && (uint64_t)n_group * 4u > r.len - r.n)) r.ok = false;
      if (r.ok) wr_skip(r, (uint32_t)n_group * 4u);
    }
    if (!r.ok || r.n != r.len) st = GPX_WS_MALFORMED;
  }
  uint32_t gid = GPX_NAME_NONE;
  GroupCtx g;
  uint8_t acc_idx = 0xffu, dst_idx = 0xffu;
  if (st == GPX_WS_OK) {
    gid = wire_name_find(W, r.p + h.id_at, h.id_len);
    st = wire_group(S, W, gid, h.version, g);
  }
  if (st == GPX_WS_OK) {
    if (h.type == GPX_PT_BATCHED_ACCEPT_REPLY) {
      acc_idx = wire_member_idx(g.ms, g.R, acceptor);
      dst_idx = wire_member_idx(g.ms, g.R, bcoord);
      if (acc_idx == 0xffu || dst_idx == 0xffu) st = GPX_WS_MALFORMED; /* acceptor / coordinator not a member */
      else if (g.ms->lane_of_idx[dst_idx] == 0xffu) st = GPX_WS_NOT_LOCAL;
    } else if (g.ms->lane_mask == 0) {
      st = GPX_WS_NOT_LOCAL;
    }
  }
  if (st == GPX_WS_OK) {
    if (h.type == GPX_PT_ACCEPT) {
      c[WD_ACC] = 1;
      const uint32_t nreq = 1u + B.n_sub;
      c[WD_BLOB] = ((nreq > 1 ? 16u * nreq : 0u) + B.val + 15u) & ~15u;
    } else if (h.type == GPX_PT_BATCHED_ACCEPT_REPLY) {
      c[WD_REP] = (uint32_t)cnt_slots;
    } else {
      c[WD_DEC] = (uint32_t)cnt_slots;
    }
  }
  if (!A.emit) {
    A.status[k] = st;
    for (int j = 0; j < WD_NCNT; j++) A.cnt[(size_t)j * A.n + k] = c[j];
    return;
  }
  if (h.type == GPX_PT_ACCEPT) {
    const uint32_t o = A.off[(size_t)WD_ACC * A.n + k], bo = A.off[(size_t)WD_BLOB * A.n + k];
    const uint32_t nreq = 1u + B.n_sub;
    uint8_t* blob = A.blob + bo;
    if (nreq == 1) {
      wire_copy(blob, r.p + q.val_at, q.val_len);
    } else { /* [nreq x gpx_batch_ent][values] as gpx_propose builds it (k_build_blobs) */
      uint32_t vo = 16u * nreq;
      gpx_batch_ent be;
      be.req_id = q.req_id;
      be.len = q.val_len;
      be.flags = (q.stop ? GPX_F_STOP : 0u) | wire_entry_bits(S, q.entry);
      wire_copy(blob, reinterpret_cast<const uint8_t*>(&be), 16);
      wire_copy(blob + vo, r.p + q.val_at, q.val_len);
      vo += q.val_len;
      WireRd rr = wr_open(r.p + B.sub_at, r.len - B.sub_at, true);
      for (uint32_t b = 0; b < B.n_sub; b++) {
        WireRd s;
        WireReq sq;
        wr_latched(rr, s, sq, nullptr);
        be.req_id = sq.req_id;
        be.len = sq.val_len;
        be.flags = (sq.stop ? GPX_F_STOP : 0u) | wire_entry_bits(S, sq.entry);
        wire_copy(blob + 16u * (1u + b), reinterpret_cast<const uint8_t*>(&be), 16);
        wire_copy(blob + vo, s.p + sq.val_at, sq.val_len);
        vo += sq.val_len;
      }
    }
    const uint32_t used = (nreq > 1 ? 16u * nreq : 0u) + B.val;
    for (uint32_t b = used; b < c[WD_BLOB]; b++) blob[b] = 0;
    gpx_accept_rec a;
    a.h.gid = gid;
    a.h.slot = slot;
    a.h.bnum = bnum;
    a.h.bcoord = bcoord;
    a.h.median_cp = median;
    a.h.flags = (uint16_t)(GPX_F_ACCEPT | (B.stop ? GPX_F_STOP : 0u));
    a.h.dst_mask = g.ms->lane_mask;
    a.h.req_id = q.req_id;
    a.payload_off = bo;
    a.payload_len = used;
    a.nreq = nreq;
    a.sender = sender;
    A.acc[o] = a;
    A.acc_key[o] = gid;
  } else if (h.type == GPX_PT_BATCHED_ACCEPT_REPLY) {
    const uint32_t o = A.off[(size_t)WD_REP * A.n + k];
    WireRd s = wr_open(r.p + slots_at, r.len - slots_at, true);
    gpx_accept_reply_rec x = wire_reply_rec(gid, bnum, bcoord, max_cp, GPX_WHO(acc_idx, dst_idx, 0u));
    for (uint32_t j = 0; j < (uint32_t)cnt_slots; j++) {
      x.slot = wr_i32(s);
      x.req_id = wr_i64(s);
      A.rep[o + j] = x;
      A.rep_key[o + j] = gid;
    }
  } else {
    const uint32_t o = A.off[(size_t)WD_DEC * A.n + k];
    WireRd s = wr_open(r.p + slots_at, r.len - slots_at, true);
    gpx_decision_rec d = wire_decision_rec(gid, bnum, bcoord, median, g.ms->lane_mask);
    for (uint32_t j = 0; j < (uint32_t)cnt_slots; j++) {
      d.slot = wr_i32(s);
      A.dec[o + j] = d;
      A.dec_key[o + j] = gid;
    }
  }
}

/* ---- REQUEST packets -> proposals (gpx_wire_decode_requests_device) ------------------------------------------------ */
enum { WQ_REQ = 0, WQ_PAY = 1, WQ_NCNT = 2 };

struct WireReqDecodeArgs {
  const uint8_t* bytes;
  const gpx_wire_ref* pkts;
  uint64_t n_bytes;
  uint32_t n;
  long long now_ms;
  uint32_t* cnt;  /* [WQ_NCNT][n]: pass 0 writes the packet's requests and payload bytes (each value padded to 16) */
  const uint32_t* off; /* [WQ_NCNT][n]: pass 1 reads their exclusive prefix sums */
  int32_t* status;
  /* pass 1: requests and meta staged in packet order, the sort keys (gids) beside them; the payload is the output */
  gpx_request_rec* req;
  gpx_wire_req_meta* meta;
  uint32_t* key;
  uint8_t* payload;
  int emit;
};

/* where a packet's requests go: staged position o and payload offset po, both advanced per request, and what the
 * packet's requests share (their gid, client handle, receiving node and the lane serving it) */
struct WireReqTo {
  uint32_t o, po, gid, client, lane;
  int32_t node;
};
/* one request: its record, meta and sort key at t.o, and the zero padding of its value to 16 bytes.  Returns where the
 * caller writes the val_len value bytes.  Args: WireReqDecodeArgs, or the JSON decoder's WireJsonReqArgs. */
template <typename Args>
__device__ __forceinline__ uint8_t* wire_put_request(const Args& A, WireReqTo& t, int64_t req_id, bool stop,
                                                     int32_t entry, uint32_t val_len, gpx_wire_req_meta m) {
  gpx_request_rec rq;
  rq.gid = t.gid;
  rq.flags = (stop ? GPX_F_STOP : 0u) | (t.lane << 8);
  rq.req_id = req_id;
  rq.payload_off = t.po;
  rq.payload_len = val_len;
  if (entry == -1) { /* IntegerMap.NULL_INT_NODE: setEntryReplica :393-403 with the call's clock */
    rq.entry_node = t.node;
    m.entry_time = A.now_ms;
  } else {
    rq.entry_node = entry;
  }
  rq.client = t.client;
  A.req[t.o] = rq;
  A.meta[t.o] = m;
  A.key[t.o] = t.gid;
  t.o++;
  uint8_t* d = A.payload + t.po;
  const uint32_t padded = (val_len + 15u) & ~15u;
  for (uint32_t b = val_len; b < padded; b++) d[b] = 0;
  t.po += padded;
  return d;
}

/* one thread per packet.  Pass 0 (emit == 0) parses and validates the packet (the request part of k_wire_decode's
 * ACCEPT rules), looks its name and receiving node up and writes its status and output sizes; pass 1 parses it again
 * and writes its requests, meta and values at the scanned offsets. */
__global__ void k_wire_req_decode(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                  const __grid_constant__ WireReqDecodeArgs A) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= A.n) return;
  if (A.emit && A.status[k] != GPX_WS_OK) return;
  const gpx_wire_ref ref = A.pkts[k];
  WireRd r;
  WireHdr h;
  int32_t st = wr_packet(A.bytes, A.n_bytes, ref, GPX_PT_BIT(GPX_PT_REQUEST), r, h);
  WireReq q;
  WireReqMore x;
  WireBatch B = {};
  if (st == GPX_WS_OK) {
    wr_request_batch(r, q, &x, B);
    if (!r.ok || r.n != r.len) st = GPX_WS_MALFORMED;
    else if (B.host_only) st = GPX_WS_UNHANDLED; /* digest mode / a response: the host's */
  }
  uint32_t gid = GPX_NAME_NONE, lane = 0;
  GroupCtx g;
  if (st == GPX_WS_OK) {
    gid = wire_name_find(W, r.p + h.id_at, h.id_len);
    st = wire_group(S, W, gid, h.version, g);
  }
  if (st == GPX_WS_OK) st = wire_recv_lane(S, g, ref.node, lane);
  if (!A.emit) {
    A.status[k] = st;
    A.cnt[k] = st == GPX_WS_OK ? 1u + B.n_sub : 0u;
    A.cnt[A.n + k] = st == GPX_WS_OK ? B.pay : 0u;
    return;
  }
  WireReqTo t = {A.off[k], A.off[A.n + k], gid, k, lane, ref.node};
  wire_copy(wire_put_request(A, t, q.req_id, q.stop, q.entry, q.val_len, x.m), r.p + q.val_at, q.val_len);
  WireRd rr = wr_open(r.p + B.sub_at, r.len - B.sub_at, true);
  for (uint32_t b = 0; b < B.n_sub; b++) {
    WireRd s;
    WireReq sq;
    WireReqMore sx;
    wr_latched(rr, s, sq, &sx);
    wire_copy(wire_put_request(A, t, sq.req_id, sq.stop, sq.entry, sq.val_len, sx.m), s.p + sq.val_at, sq.val_len);
  }
}

/* launch glue of the host side (gpx_wire_host.inc) */
__global__ void k_wire_iota(uint32_t* p, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}
/* tot[j] = the total of counter row j of [rows][n] from its exclusive prefix sums */
__global__ void k_wire_totals(const uint32_t* cnt, const uint32_t* off, uint32_t n, uint32_t rows, uint32_t* tot) {
  const uint32_t j = threadIdx.x;
  if (j < rows) tot[j] = off[(size_t)j * n + n - 1] + cnt[(size_t)j * n + n - 1];
}

/* records (or their indices) into the order of a stable sort: dst[i] = src[perm[i]] */
template <typename T>
__global__ void k_wire_gather(const T* src, const uint32_t* perm, uint32_t n, T* dst) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[perm[i]];
}

/* ---- encode ---------------------------------------------------------------------------------------------------- */
struct WireEncodeArgs {
  const void* recs;     /* gpx_accept_reply_rec[n] or gpx_decision_rec[n] */
  uint32_t n;
  uint32_t n_lanes;     /* replies: record i * n_lanes + l belongs to lane l */
  uint8_t* rstatus;     /* [n] GPX_WE_* per record */
  uint32_t* key;        /* [n] sort key: (lane, gid) / gid, GPX_WIRE_NOKEY if not encoded */
  const uint32_t* perm; /* [n] record indices in stable key order (GPX_WIRE_NOKEY keys last) */
  const uint32_t* skey; /* [n] the keys in that order */
  uint32_t* cnt;        /* [2][n] pass 0, per sorted position that starts a run: packet bytes, index entries */
  const uint32_t* off;  /* [2][n] their exclusive prefix sums */
  uint8_t* out;
  gpx_wire_ref* refs;
  int emit;
  const uint32_t* n_ptr; /* decisions: records [*n_ptr, n) are not read and get no rstatus (device count); null = n */
};

/* where a reply that is neither void nor a NACK goes: GPX_WE_VOID (its group is gone, or a member index is out of
 * range), GPX_WE_LOCAL (a local lane serves its destination: SHORT_CIRCUIT_LOCAL), GPX_WE_NO_NAME, else GPX_WE_SENT.
 * The JSON encoder (gpx_wire_json_enc.cuh) routes a NACK by the same rule. */
__device__ __forceinline__ uint8_t wire_reply_route(const DevState& S, const WireNames& W, const gpx_accept_reply_rec& x,
                                                    const GroupCtx& g) {
  if (!g.live || GPX_WHO_DST(x.who) >= g.R || GPX_WHO_ACC(x.who) >= g.R) return GPX_WE_VOID;
  if (g.ms->lane_of_idx[GPX_WHO_DST(x.who)] != 0xffu) return GPX_WE_LOCAL;
  if (W.slot == nullptr || W.slot[x.gid] == GPX_NAME_NONE) return GPX_WE_NO_NAME;
  return GPX_WE_SENT;
}
/* one thread per record: what happens to it and its sort key */
__global__ void k_wire_enc_keys_replies(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                        const __grid_constant__ WireEncodeArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const gpx_accept_reply_rec x = reinterpret_cast<const gpx_accept_reply_rec*>(A.recs)[i];
  const uint32_t fl = GPX_WHO_FLAGS(x.who), lane = i % A.n_lanes;
  uint8_t st;
  const GroupCtx g = group_ctx(S, x.gid);
  if (fl & GPX_F_VOID) st = GPX_WE_VOID;
  else if (fl & GPX_F_NACK) st = GPX_WE_NACK; /* allPositiveAcceptReplies :423-430: never coalesced */
  else st = wire_reply_route(S, W, x, g);
  A.rstatus[i] = st;
  A.key[i] = st == GPX_WE_SENT ? lane * S.G + x.gid : GPX_WIRE_NOKEY;
}
/* a decision or an ACCEPT for every member: GPX_WE_VOID (a void record, or its group is gone), GPX_WE_LOCAL (every
 * member is a local lane), GPX_WE_NO_NAME, else GPX_WE_SENT */
__device__ __forceinline__ uint8_t wire_enc_status(const DevState& S, const WireNames& W, uint32_t gid, bool void_rec) {
  const GroupCtx g = group_ctx(S, gid);
  if (void_rec || !g.live) return GPX_WE_VOID;
  if (wire_popc(g.ms->lane_mask) >= g.R) return GPX_WE_LOCAL;
  if (W.slot == nullptr || W.slot[gid] == GPX_NAME_NONE) return GPX_WE_NO_NAME;
  return GPX_WE_SENT;
}
__global__ void k_wire_enc_keys_decisions(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                          const __grid_constant__ WireEncodeArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  if (A.n_ptr && i >= *A.n_ptr) { /* past the device count: sorts last, never encoded */
    A.key[i] = GPX_WIRE_NOKEY;
    return;
  }
  const gpx_decision_rec d = reinterpret_cast<const gpx_decision_rec*>(A.recs)[i];
  const uint8_t st = wire_enc_status(S, W, d.gid, d.flags & GPX_F_VOID);
  A.rstatus[i] = st;
  A.key[i] = st == GPX_WE_SENT ? d.gid : GPX_WIRE_NOKEY;
}

__device__ __forceinline__ void ww_i32(uint8_t* p, int32_t v) {
  const uint32_t u = (uint32_t)v;
  p[0] = (uint8_t)(u >> 24);
  p[1] = (uint8_t)(u >> 16);
  p[2] = (uint8_t)(u >> 8);
  p[3] = (uint8_t)u;
}
__device__ __forceinline__ void ww_i64(uint8_t* p, int64_t v) {
  ww_i32(p, (int32_t)(uint32_t)((uint64_t)v >> 32));
  ww_i32(p + 4, (int32_t)(uint32_t)(uint64_t)v);
}
/* PaxosPacket.toBytes :459-476; returns the bytes written */
__device__ __forceinline__ uint32_t ww_header(uint8_t* p, int32_t type, const WireNames& W, uint32_t gid) {
  const uint8_t* m = W.name + (size_t)gid * GPX_NAME_BYTES;
  ww_i32(p, GPX_PT_PAXOS_PACKET);
  ww_i32(p + 4, type);
  ww_i32(p + 8, W.version[gid]);
  p[12] = m[0];
  wire_copy(p + 13, m + 1, m[0]);
  return 13u + m[0];
}

/* the run of sorted positions [p, end) that share the key and ballot of position p; false if p does not start one */
template <typename T>
__device__ __forceinline__ bool wire_run(const WireEncodeArgs& A, uint32_t p, uint32_t& end) {
  const T* recs = reinterpret_cast<const T*>(A.recs);
  const uint32_t key = A.skey[p];
  if (key == GPX_WIRE_NOKEY) return false;
  const T x = recs[A.perm[p]];
  if (p > 0 && A.skey[p - 1] == key) {
    const T y = recs[A.perm[p - 1]];
    if (y.bnum == x.bnum && y.bcoord == x.bcoord) return false;
  }
  end = p + 1;
  while (end < A.n && A.skey[end] == key) {
    const T y = recs[A.perm[end]];
    if (y.bnum != x.bnum || y.bcoord != x.bcoord) break;
    end++;
  }
  return true;
}

/* the run's distinct slots in ascending signed order (TreeMap / TreeSet): each(k, slot, bi) for the k-th of them, bi =
 * sorted position of the entry that wins a repeated slot (the last put).  Returns the number of distinct slots. */
template <typename T, typename Each>
__device__ __forceinline__ uint32_t wire_slots_each(const WireEncodeArgs& A, uint32_t p, uint32_t end, Each each) {
  const T* recs = reinterpret_cast<const T*>(A.recs);
  uint32_t n = 0;
  bool have = false;
  int32_t prev = 0;
  for (;;) { /* selection: the smallest slot above the previous one, O(run^2) -- runs are a window's worth */
    bool found = false;
    int32_t best = 0;
    uint32_t bi = 0;
    for (uint32_t q = p; q < end; q++) {
      const int32_t s = recs[A.perm[q]].slot;
      if (have && s <= prev) continue;
      if (!found || s <= best) { /* s == best: the same slot again, the later record wins */
        best = s;
        bi = q;
        found = true;
      }
    }
    if (!found) break;
    each(n, best, bi);
    n++;
    have = true;
    prev = best;
  }
  return n;
}
/* wire_slots_each writing the slots (and a reply's requestIDs) as big-endian words; out == nullptr only counts */
template <typename T, bool WITH_REQ>
__device__ __forceinline__ uint32_t wire_slots(const WireEncodeArgs& A, uint32_t p, uint32_t end, uint8_t* out) {
  const T* recs = reinterpret_cast<const T*>(A.recs);
  return wire_slots_each<T>(A, p, end, [&](uint32_t n, int32_t best, uint32_t bi) {
    if (out) {
      uint8_t* o = out + (size_t)n * (WITH_REQ ? 12u : 4u);
      ww_i32(o, best);
      if (WITH_REQ) ww_i64(o + 4, reinterpret_cast<const gpx_accept_reply_rec*>(recs)[A.perm[bi]].req_id);
    }
  });
}

/* one thread per sorted position; a position that starts a (lane, gid, ballot) run writes one BatchedAcceptReply
 * (BatchedAcceptReply(AcceptReplyPacket) :53-58 takes the header of the first reply, addAcceptReply :179-184 adds
 * slot -> requestID) addressed to the ballot's coordinator */
__global__ void k_wire_enc_replies(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                   const __grid_constant__ WireEncodeArgs A) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n) return;
  uint32_t end = 0;
  const bool head = wire_run<gpx_accept_reply_rec>(A, p, end);
  if (!A.emit) {
    uint32_t bytes = 0;
    if (head) {
      const uint32_t gid = reinterpret_cast<const gpx_accept_reply_rec*>(A.recs)[A.perm[p]].gid;
      bytes = 13u + W.name[(size_t)gid * GPX_NAME_BYTES] + 29u + 4u +
              12u * wire_slots<gpx_accept_reply_rec, true>(A, p, end, nullptr);
    }
    A.cnt[p] = bytes;
    A.cnt[A.n + p] = head ? 1u : 0u;
    return;
  }
  if (!head) return;
  const gpx_accept_reply_rec x = reinterpret_cast<const gpx_accept_reply_rec*>(A.recs)[A.perm[p]];
  const MsetInfo* ms = group_ctx(S, x.gid).ms;
  uint8_t* o = A.out + A.off[p];
  uint32_t b = ww_header(o, GPX_PT_BATCHED_ACCEPT_REPLY, W, x.gid);
  ww_i32(o + b, ms->nodes[GPX_WHO_ACC(x.who)]);
  ww_i32(o + b + 4, x.bnum);
  ww_i32(o + b + 8, x.bcoord);
  ww_i32(o + b + 12, x.slot);
  ww_i32(o + b + 16, x.max_cp);
  ww_i64(o + b + 20, x.req_id);
  o[b + 28] = 0; /* undigestRequest */
  b += 29;
  const uint32_t ns = wire_slots<gpx_accept_reply_rec, true>(A, p, end, o + b + 4);
  ww_i32(o + b, (int32_t)ns);
  b += 4 + 12u * ns;
  gpx_wire_ref r;
  r.off = A.off[p];
  r.len = b;
  r.gid = x.gid;
  r.node = ms->nodes[GPX_WHO_DST(x.who)];
  A.refs[A.off[A.n + p]] = r;
}

/* the packet of sorted position p (len bytes at A.off[p]) indexed once per member node of g that no local lane serves,
 * from index A.off[A.n + p] on; pass 0 counts g.R - wire_popc(g.ms->lane_mask) of them */
__device__ __forceinline__ void wire_refs_remote(const WireEncodeArgs& A, uint32_t p, const GroupCtx& g, uint32_t gid,
                                                 uint32_t len) {
  uint32_t ri = A.off[A.n + p];
  for (uint32_t m = 0; m < g.R; m++) {
    if (g.ms->lane_of_idx[m] != 0xffu) continue;
    gpx_wire_ref r;
    r.off = A.off[p];
    r.len = len;
    r.gid = gid;
    r.node = g.ms->nodes[m];
    A.refs[ri++] = r;
  }
}

/* the wrap-aware maximum medianCheckpointedSlot of the decision run [p, end) (BatchedCommit.addCommit :113-121) */
__device__ __forceinline__ int32_t wire_run_median(const WireEncodeArgs& A, uint32_t p, uint32_t end) {
  const gpx_decision_rec* recs = reinterpret_cast<const gpx_decision_rec*>(A.recs);
  int32_t median = recs[A.perm[p]].median_cp;
  for (uint32_t q = p + 1; q < end; q++) {
    const int32_t m = recs[A.perm[q]].median_cp;
    if (jsub(m, median) > 0) median = m;
  }
  return median;
}

/* one thread per sorted position; a position that starts a (gid, ballot) run writes one BatchedCommit
 * (PaxosPacketBatcher.fuseBatchedCommits :389-417, BatchedCommit.addCommit :113-121: medianCheckpointedSlot is the
 * wrap-aware maximum, gpx_wire_fuse_commits' rule), stored once and indexed once per member node that no local lane
 * serves */
__global__ void k_wire_enc_decisions(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                     const __grid_constant__ WireEncodeArgs A) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n) return;
  uint32_t end = 0;
  const bool head = wire_run<gpx_decision_rec>(A, p, end);
  const gpx_decision_rec* recs = reinterpret_cast<const gpx_decision_rec*>(A.recs);
  const GroupCtx g = group_ctx(S, head ? recs[A.perm[p]].gid : 0u);
  const uint32_t n_remote = head ? g.R - wire_popc(g.ms->lane_mask) : 0u;
  if (!A.emit) {
    uint32_t bytes = 0;
    if (head) {
      const uint32_t gid = recs[A.perm[p]].gid;
      bytes = 13u + W.name[(size_t)gid * GPX_NAME_BYTES] + 12u + 4u +
              4u * wire_slots<gpx_decision_rec, false>(A, p, end, nullptr) + 4u + 4u * g.R;
    }
    A.cnt[p] = bytes;
    A.cnt[A.n + p] = n_remote;
    return;
  }
  if (!head) return;
  const gpx_decision_rec d = recs[A.perm[p]];
  const int32_t median = wire_run_median(A, p, end);
  uint8_t* o = A.out + A.off[p];
  uint32_t b = ww_header(o, GPX_PT_BATCHED_COMMIT, W, d.gid);
  ww_i32(o + b, d.bnum);
  ww_i32(o + b + 4, d.bcoord);
  ww_i32(o + b + 8, median);
  b += 12;
  const uint32_t ns = wire_slots<gpx_decision_rec, false>(A, p, end, o + b + 4);
  ww_i32(o + b, (int32_t)ns);
  b += 4 + 4u * ns;
  ww_i32(o + b, (int32_t)g.R);
  b += 4;
  for (uint32_t m = 0; m < g.R; m++, b += 4) ww_i32(o + b, g.ms->nodes[m]);
  wire_refs_remote(A, p, g, d.gid, b);
}

/* ---- ACCEPTs -> AcceptPacket bytes (gpx_wire_encode_accepts_device) --------------------------------------------------- */
struct WireAccArgs {
  const uint32_t* head;          /* [n] request index that starts ACCEPT k (gpx_propose_device_heads) */
  const gpx_request_rec* reqs;   /* [n_reqs] */
  const gpx_wire_req_meta* meta; /* [n_reqs] */
  uint32_t n_reqs;
  const uint8_t* payload;        /* the request arena: bodies at reqs[q].payload_off */
};

/* one thread per ACCEPT: what happens to it and its sort key (the gid); past the device count: sorts last, unread */
__global__ void k_wire_enc_keys_accepts(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                        const __grid_constant__ WireEncodeArgs A, const __grid_constant__ WireAccArgs X) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  if (A.n_ptr && i >= *A.n_ptr) {
    A.key[i] = GPX_WIRE_NOKEY;
    return;
  }
  const gpx_accept_rec a = reinterpret_cast<const gpx_accept_rec*>(A.recs)[i];
  uint8_t st = wire_enc_status(S, W, a.h.gid, a.h.flags & GPX_F_VOID);
  if (st == GPX_WE_SENT) {
    const uint32_t q = X.head[i];
    if (a.nreq == 0 || q >= X.n_reqs || a.nreq > X.n_reqs - q || X.reqs[q].gid != a.h.gid) st = GPX_WE_BAD_HEAD;
  }
  A.rstatus[i] = st;
  A.key[i] = st == GPX_WE_SENT ? a.h.gid : GPX_WIRE_NOKEY;
}

/* RequestPacket.toBytes :819-949 of one request without batched requests (n_batched written by the caller's count):
 * its record, its wire meta and the arena its value lies in (at rq.payload_off).  Shared with the journal frames
 * (gpx_journal.cuh) */
__device__ __forceinline__ uint32_t ww_request_rec(uint8_t* p, int32_t type, const WireNames& W, uint32_t gid,
                                                   const gpx_request_rec rq, const gpx_wire_req_meta m,
                                                   const uint8_t* payload, uint32_t n_batched) {
  uint32_t b = ww_header(p, type, W, gid);
  ww_i64(p + b, rq.req_id);
  p[b + 8] = (rq.flags & GPX_F_STOP) ? 1u : 0u;
  b += 9;
  for (int j = 0; j < 4; j++) p[b + j] = m.client_port ? m.client_ip[j] : 0u;
  p[b + 4] = (uint8_t)(m.client_port >> 8);
  p[b + 5] = (uint8_t)m.client_port;
  for (int j = 0; j < 4; j++) p[b + 6 + j] = m.listen_port ? m.listen_ip[j] : 0u;
  p[b + 10] = (uint8_t)(m.listen_port >> 8);
  p[b + 11] = (uint8_t)m.listen_port;
  b += 12;
  ww_i32(p + b, rq.entry_node);
  ww_i64(p + b + 4, m.entry_time);
  p[b + 12] = (m.flags & GPX_RM_RETURN_VALUE) ? 1u : 0u;
  ww_i32(p + b + 13, m.forward_count);
  p[b + 17] = (m.flags & GPX_RM_BROADCASTED) ? 1u : 0u;
  ww_i32(p + b + 18, 0); /* digest */
  ww_i32(p + b + 22, (int32_t)rq.payload_len);
  b += 26;
  wire_copy(p + b, payload + rq.payload_off, rq.payload_len);
  b += rq.payload_len;
  ww_i32(p + b, 0); /* responseValue */
  ww_i32(p + b + 4, (int32_t)n_batched);
  return b + 8;
}
/* the bytes ww_request_rec writes for a value of val_len bytes */
__device__ __forceinline__ uint32_t ww_request_bytes(const WireNames& W, uint32_t gid, uint32_t val_len) {
  return 13u + W.name[(size_t)gid * GPX_NAME_BYTES] + 55u + val_len;
}
/* request q of the ACCEPTs' requests */
__device__ __forceinline__ uint32_t ww_request(uint8_t* p, int32_t type, const WireNames& W, uint32_t gid,
                                               const WireAccArgs& X, uint32_t q, uint32_t n_batched) {
  return ww_request_rec(p, type, W, gid, X.reqs[q], X.meta[q], X.payload, n_batched);
}
/* requests q0 .. q0 + n - 1 as one packet: the first of type `type`, the others its latched REQUESTs
 * ({int length}{REQUEST packet} :929-936); returns the bytes written */
__device__ __forceinline__ uint32_t ww_requests(uint8_t* p, int32_t type, const WireNames& W, uint32_t gid,
                                                const WireAccArgs& X, uint32_t q0, uint32_t n) {
  uint32_t b = ww_request(p, type, W, gid, X, q0, n - 1u);
  for (uint32_t q = q0 + 1; q < q0 + n; q++) {
    const uint32_t l = ww_request(p + b + 4, GPX_PT_REQUEST, W, gid, X, q, 0u);
    ww_i32(p + b, (int32_t)l);
    b += 4u + l;
  }
  return b;
}
/* the bytes ww_requests writes: per request the header, 55 fixed bytes and the value, and 4 per latched one */
__device__ __forceinline__ uint32_t wire_requests_bytes(const WireNames& W, uint32_t gid, const gpx_request_rec* reqs,
                                                        uint32_t q0, uint32_t n) {
  uint32_t bytes = 0;
  for (uint32_t q = q0; q < q0 + n; q++)
    bytes += 13u + W.name[(size_t)gid * GPX_NAME_BYTES] + 55u + reqs[q].payload_len + (q > q0 ? 4u : 0u);
  return bytes;
}

/* one thread per sorted position; every encoded ACCEPT is one AcceptPacket (AcceptPacket.toBytes :95-138), stored once
 * and indexed once per member node that no local lane serves */
__global__ void k_wire_enc_accepts(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                                   const __grid_constant__ WireEncodeArgs A, const __grid_constant__ WireAccArgs X) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= A.n) return;
  const bool sent = A.skey[p] != GPX_WIRE_NOKEY;
  const gpx_accept_rec* recs = reinterpret_cast<const gpx_accept_rec*>(A.recs);
  const uint32_t i = sent ? A.perm[p] : 0u;
  if (!A.emit) {
    uint32_t bytes = 0, n_remote = 0;
    if (sent) {
      const gpx_accept_rec a = recs[i];
      const GroupCtx g = group_ctx(S, a.h.gid);
      bytes = wire_requests_bytes(W, a.h.gid, X.reqs, X.head[i], a.nreq) + 22u;
      n_remote = g.R - wire_popc(g.ms->lane_mask);
    }
    A.cnt[p] = bytes;
    A.cnt[A.n + p] = n_remote;
    return;
  }
  if (!sent) return;
  const gpx_accept_rec a = recs[i];
  const GroupCtx g = group_ctx(S, a.h.gid);
  uint8_t* o = A.out + A.off[p];
  uint32_t b = ww_requests(o, GPX_PT_ACCEPT, W, a.h.gid, X, X.head[i], a.nreq);
  ww_i32(o + b, a.h.slot);
  ww_i32(o + b + 4, a.h.bnum);
  ww_i32(o + b + 8, a.h.bcoord);
  o[b + 12] = 0; /* recovery */
  ww_i32(o + b + 13, a.h.median_cp);
  o[b + 17] = 0; /* noCoalesce */
  ww_i32(o + b + 18, a.sender);
  b += 22;
  wire_refs_remote(A, p, g, a.h.gid, b);
}
