/*
 * rc_emu.cpp -- the response cache's sequences (rc_put, rc_match of gigapaxos_b200/csrc/gpx_wire_seq.h) over its
 * kernels (gpx_respcache.cuh, the source the GPU runs) on the CPU executor of wire_exec.h.  The table, the generations
 * and the name slots are arrays the test hands in.  Test infrastructure only.
 */
#include "wire_exec.h"

/* slot = nullptr: no name state (gen is then not read) */
static RcTable table(RcCell* cell, uint32_t mask, uint32_t G, int64_t timeout_ms, const uint32_t* gen,
                     const uint32_t* slot) {
  RcTable T;
  T.cell = cell;
  T.mask = mask;
  T.G = G;
  T.timeout_ms = timeout_ms;
  T.gen = slot ? gen : nullptr;
  T.slot = slot;
  return T;
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

/* gpx_response_cache_put_device */
extern "C" int emu_rc_put(RcCell* cell, uint32_t mask, uint32_t G, int64_t timeout_ms, const uint32_t* gen,
                          const uint32_t* slot, const gpx_rc_key* keys, uint32_t n, int64_t now_ms, uint32_t block) {
  EmuExec ex{block};
  EmuCall call;
  return rc_put(ex, call, &ex.buf, &ex.bytes, table(cell, mask, G, timeout_ms, gen, slot), n, keys, now_ms);
}

/* gpx_response_cache_match_device */
extern "C" int emu_rc_match(const RcCell* cell, uint32_t mask, uint32_t G, int64_t timeout_ms, const uint32_t* gen,
                            const uint32_t* slot, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta,
                            uint32_t n, int64_t now_ms, int32_t* hit, gpx_request_rec* out_reqs,
                            gpx_wire_req_meta* out_meta, uint32_t* n_out, uint32_t block) {
  EmuExec ex{block};
  EmuCall call;
  return rc_match(ex, call, &ex.buf, &ex.bytes, table(const_cast<RcCell*>(cell), mask, G, timeout_ms, gen, slot), n,
                  reqs, meta, now_ms, hit, out_reqs, out_meta, n_out);
}
