/*
 * p1b_emu.cpp -- k_prepare_tally (gigapaxos_b200/csrc/gpx_phase1b.cuh, the source the GPU runs) compiled for the host
 * over cuda_emu.h, driven by the product's own host sequence (prepare_replies in gpx_state_seq.h) on the CPU executor,
 * in the world of state_exec.h.  Outputs and state are left where the kernel wrote them.  Test infrastructure only.
 */
#include "state_exec.h"

/* gpx_handle_prepare_replies; returns the kernel launches the call counted, or its GPX_* error */
extern "C" int emu_prepare_tally(uint32_t G, uint32_t L, uint32_t W, uint32_t Rcap, uint32_t R, const int32_t* members,
                                 const int32_t* lane_node, const uint8_t* live, int32_t* coord_row, uint32_t* acc_aux,
                                 int32_t* node_slots, int32_t* prop_win, uint32_t n, const gpx_election_rec* els,
                                 uint32_t n_reply_recs, const gpx_prepare_reply_rec* replies, gpx_election_out* out,
                                 uint32_t block) {
  EmuWorld w(G, L, W, Rcap, R, members, lane_node, live, block);
  if (!w.ok) return -100;
  w.S.acc_aux = acc_aux;
  w.S.coord_row = reinterpret_cast<int4*>(coord_row);
  w.S.node_slots = node_slots;
  w.S.prop_win = reinterpret_cast<int4*>(prop_win);
  return w.done(prepare_replies(w.ex, w.env(), n, els, n_reply_recs, replies, out));
}
