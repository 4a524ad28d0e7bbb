/*
 * logfind_emu.cpp -- k_log_dir / k_log_scan / k_log_hits and k_log_gather (gigapaxos_b200/csrc/gpx_logfind.cuh, the
 * source the GPU runs) compiled for the host over cuda_emu.h, driven by the product's own host sequences (log_find and
 * log_gather in gpx_state_seq.h) on the CPU executor.  The caller hands in one lane's ring as the device holds it
 * (ring_cap bytes, positions taken modulo ring_cap) and the head.  Test infrastructure only.
 */
#include "state_exec.h"

/* the head the engine reads once the rounds are done */
struct EmuHead {
  uint64_t head;
  int begin() { return GPX_OK; }
};

/* gpx_log_find; k_log_scan runs grid x block threads.  Returns 1 (k_log_dir's launch) or the GPX_* error. */
extern "C" int emu_log_find(uint8_t* ring, uint64_t ring_cap, uint64_t head, uint64_t from, uint32_t lane, uint32_t n,
                            const gpx_log_want* wants, gpx_log_hit* hits, uint32_t grid, uint32_t block) {
  EmuWorld w(0, lane + 1, 0, 0, 0, nullptr, nullptr, nullptr, block);
  if (!w.ok || (ring_cap & (ring_cap - 1))) return -100;
  w.ring(lane, ring, ring_cap, head);
  EmuCall call;
  return w.done(log_find(w.ex, call, w.env(), lane, from, n, wants, hits, grid * block));
}

/* gpx_log_gather into out[out_bytes]; returns 0 or the GPX_* error */
extern "C" int emu_log_gather(uint8_t* ring, uint64_t ring_cap, uint64_t head, uint32_t lane, uint32_t n,
                              const gpx_log_range* ranges, uint8_t* out, uint64_t out_bytes, uint32_t block) {
  EmuWorld w(0, lane + 1, 0, 0, 0, nullptr, nullptr, nullptr, block);
  if (!w.ok || (ring_cap & (ring_cap - 1))) return -100;
  w.ring(lane, ring, ring_cap, head);
  EmuHead call{head};
  return w.done(log_gather(w.ex, call, w.env(), lane, n, ranges, out, out_bytes));
}
