/*
 * pause_emu.cpp -- k_pause_groups, k_select_groups, k_missing_decisions and k_clear_flags (gigapaxos_b200/csrc/
 * gpx_pause.cuh, the source the GPU runs) compiled for the host over cuda_emu.h, driven by the product's own host
 * sequences (gpx_state_seq.h) on the CPU executor, in the world of state_exec.h.  Each returns the kernel launches the
 * call counted, or its GPX_* error.  Test infrastructure only.
 */
#include "state_exec.h"

static void planes(EmuWorld& w, int journaling, int32_t* acc_row, uint32_t* acc_aux, int32_t* acc_win,
                   int32_t* coord_row, int32_t* node_slots) {
  w.S.journaling = journaling;
  w.S.acc_row = reinterpret_cast<int4*>(acc_row);
  w.S.acc_aux = acc_aux;
  w.S.acc_win = reinterpret_cast<int4*>(acc_win);
  w.S.coord_row = reinterpret_cast<int4*>(coord_row);
  w.S.node_slots = node_slots;
}

/* gpx_pause_groups up to the rows' version and name hash, which the engine keeps on the host */
extern "C" int emu_pause_groups(uint32_t G, uint32_t L, uint32_t W, uint32_t Rcap, uint32_t R, const int32_t* members,
                                const int32_t* lane_node, const uint8_t* live, int journaling, int32_t* acc_row,
                                uint32_t* acc_aux, int32_t* acc_win, int32_t* coord_row, int32_t* node_slots, uint32_t n,
                                const uint32_t* gids, gpx_row* rows, uint8_t* paused, uint32_t block) {
  EmuWorld w(G, L, W, Rcap, R, members, lane_node, live, block);
  if (!w.ok) return -100;
  planes(w, journaling, acc_row, acc_aux, acc_win, coord_row, node_slots);
  return w.done(pause_groups(w.ex, w.env(), n, gids, rows, paused));
}

extern "C" int emu_select_groups(uint32_t G, uint32_t L, uint32_t W, uint32_t Rcap, uint32_t R, const int32_t* members,
                                 const int32_t* lane_node, const uint8_t* live, int journaling, int32_t* acc_row,
                                 uint32_t* acc_aux, int32_t* acc_win, int32_t* coord_row, uint32_t lane, uint32_t mask,
                                 uint32_t value, uint32_t* gids, uint32_t cap, uint32_t* n_found, uint32_t block) {
  EmuWorld w(G, L, W, Rcap, R, members, lane_node, live, block);
  if (!w.ok) return -100;
  planes(w, journaling, acc_row, acc_aux, acc_win, coord_row, nullptr);
  return w.done(select_groups(w.ex, w.env(), lane, mask, value, gids, cap, n_found));
}

extern "C" int emu_missing_decisions(uint32_t G, uint32_t L, uint32_t W, uint32_t R, const int32_t* members,
                                     const int32_t* lane_node, const uint8_t* live, int journaling, int32_t* acc_row,
                                     uint32_t* acc_aux, int32_t* acc_win, int32_t* coord_row, uint32_t lane, uint32_t n,
                                     const uint32_t* gids, int32_t size_limit, int32_t too_much_gap, gpx_missing_rec* out,
                                     uint32_t block) {
  EmuWorld w(G, L, W, R, R, members, lane_node, live, block);
  if (!w.ok) return -100;
  planes(w, journaling, acc_row, acc_aux, acc_win, coord_row, nullptr);
  return w.done(missing_decisions(w.ex, w.env(), lane, n, gids, size_limit, too_much_gap, out));
}

extern "C" int emu_clear_group_flags(uint32_t G, uint32_t L, uint32_t W, uint32_t R, const int32_t* members,
                                     const int32_t* lane_node, const uint8_t* live, uint32_t* acc_aux, uint32_t lane,
                                     uint32_t n, const uint32_t* gids, uint32_t mask, uint32_t block) {
  EmuWorld w(G, L, W, R, R, members, lane_node, live, block);
  if (!w.ok) return -100;
  w.S.acc_aux = acc_aux;
  return w.done(clear_group_flags(w.ex, w.env(), lane, n, gids, mask));
}
