/*
 * rc_emu.cpp -- the response cache's kernels (gigapaxos_b200/csrc/gpx_respcache.cuh, the source the GPU runs) compiled
 * for the host over cuda_emu.h.  The table, the generations and the name slots are arrays the test hands in; the
 * stable sorts and the scan that gpx_respcache_host.inc does with CUB are done here with the standard library.  Test
 * infrastructure only.
 */
#include "cuda_emu.h"

template <class T>
static inline T atomicCAS(T* p, T cmp, T v) { /* gpx_wire_dev.cuh's name table; never called here */
  T old = *p;
  if (old == cmp) *p = v;
  return old;
}

#include <numeric>
#include <vector>

#include "gpx_respcache.cuh"

static RcTable table(RcCell* cell, uint32_t mask, uint32_t G, int64_t timeout_ms, const uint32_t* gen,
                     const uint32_t* slot) {
  RcTable T;
  T.cell = cell;
  T.mask = mask;
  T.G = G;
  T.timeout_ms = timeout_ms;
  T.gen = gen;
  T.slot = slot;
  return T;
}

/* perm: indices in the stable order of key; sorted: the keys in that order */
static void stable_sort(const std::vector<uint32_t>& key, std::vector<uint32_t>& perm, std::vector<uint32_t>& sorted) {
  perm.resize(key.size());
  std::iota(perm.begin(), perm.end(), 0u);
  std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  sorted.resize(key.size());
  for (size_t j = 0; j < key.size(); j++) sorted[j] = key[perm[j]];
}

extern "C" uint32_t emu_rc_cell_bytes(void) { return sizeof(RcCell); }

extern "C" uint64_t emu_rc_hash(uint32_t gid, uint32_t gen, int64_t req_id, uint32_t ip, uint16_t port) {
  return rc_hash(gid, gen, req_id, ip, port);
}

extern "C" void emu_rc_gen_bump(uint32_t* gen, const uint32_t* gids, uint32_t n, uint32_t block) {
  NameSetArgs A;
  A.gids = gids;
  A.n = n;
  emu_launch(k_rc_gen_bump, (n + block - 1) / block, block, gen, A);
}

/* gpx_response_cache_put_device without the copies; slot = nullptr: no name state (gen is then not read) */
extern "C" int emu_rc_put(RcCell* cell, uint32_t mask, uint32_t G, int64_t timeout_ms, const uint32_t* gen,
                          const uint32_t* slot, const gpx_rc_key* keys, uint32_t n, int64_t now_ms, uint32_t block) {
  if (n == 0) return 0;
  const RcTable T = table(cell, mask, G, timeout_ms, slot ? gen : nullptr, slot);
  std::vector<uint32_t> bucket(n), kgen(n), perm, sorted;
  uint32_t bad = 0;
  RcPutArgs A;
  memset(&A, 0, sizeof A);
  A.keys = keys;
  A.n = n;
  A.now_ms = now_ms;
  A.bucket = bucket.data();
  A.gen = kgen.data();
  A.bad = &bad;
  emu_launch(k_rc_put_keys, (n + block - 1) / block, block, T, A);
  if (bad) return GPX_EINVAL;
  stable_sort(bucket, perm, sorted);
  A.perm = perm.data();
  A.sbucket = sorted.data();
  emu_launch(k_rc_put, (n + block - 1) / block, block, T, A);
  return 0;
}

/* gpx_response_cache_match_device without the copies */
extern "C" int emu_rc_match(const RcCell* cell, uint32_t mask, uint32_t G, int64_t timeout_ms, const uint32_t* gen,
                            const uint32_t* slot, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta,
                            uint32_t n, int64_t now_ms, int32_t* hit, gpx_request_rec* out_reqs,
                            gpx_wire_req_meta* out_meta, uint32_t* n_out, uint32_t block) {
  *n_out = 0;
  if (n == 0) return 0;
  const RcTable T = table(const_cast<RcCell*>(cell), mask, G, timeout_ms, slot ? gen : nullptr, slot);
  std::vector<uint32_t> client(n), perm, sorted, dup(n), miss(n), off(n);
  for (uint32_t q = 0; q < n; q++) client[q] = reqs[q].client;
  stable_sort(client, perm, sorted);
  RcMatchArgs A;
  memset(&A, 0, sizeof A);
  A.reqs = reqs;
  A.meta = meta;
  A.n = n;
  A.now_ms = now_ms;
  A.perm = perm.data();
  A.sclient = sorted.data();
  A.dup = dup.data();
  A.hit = hit;
  A.miss = miss.data();
  A.off = off.data();
  A.out_reqs = out_reqs;
  A.out_meta = out_meta;
  const uint32_t g = (n + block - 1) / block;
  emu_launch(k_rc_dups, g, block, A);
  emu_launch(k_rc_match, g, block, T, A);
  uint32_t s = 0;
  for (uint32_t q = 0; q < n; q++) {
    off[q] = s;
    s += miss[q];
  }
  emu_launch(k_rc_scatter, g, block, A);
  *n_out = s;
  return 0;
}
