/*
 * state_exec.h -- the world the group-state and log-index sequences of gigapaxos_b200/csrc/gpx_state_seq.h run on in
 * the CPU tests: a DevState around the state arrays a test hands in (laid out as DevState describes them: [L][G] rows,
 * [L][W][G] windows, [L][Rcap][G] nodeSlotNumbers), every group in one member set, and the CPU executor of
 * wire_exec.h.  Test infrastructure only.
 */
#pragma once
#include "wire_exec.h"

#include "gpx_state_seq.h"

struct EmuWorld {
  bool ok; /* the sizes fit DevState and MsetInfo */
  MsetInfo ms;
  std::vector<uint32_t> meta;
  std::vector<unsigned long long> ctr, log_pos;
  DevState S;
  EmuExec ex;

  /* G groups over L lanes; the R members[] of the one member set, lane l serving lane_node[l]; live[g] (null: none) */
  EmuWorld(uint32_t G, uint32_t L, uint32_t W, uint32_t Rcap, uint32_t R, const int32_t* members,
           const int32_t* lane_node, const uint8_t* live, uint32_t block)
      : ok(R <= GPX_MAX_GROUP_SIZE && L <= GPX_MAX_LANES && block > 0), meta(G),
        ctr((size_t)GPX_CTR_STRIPES * C_NCTR, 0ull), log_pos((size_t)2 * GPX_MAX_LANES * 2, 0ull), ex{block} {
    memset(&ms, 0, sizeof ms);
    memset(ms.lane_of_idx, 0xff, sizeof ms.lane_of_idx);
    memset(ms.idx_of_lane, 0xff, sizeof ms.idx_of_lane);
    ms.R = (uint8_t)R;
    for (uint32_t m = 0; ok && m < R; m++) {
      ms.nodes[m] = members[m];
      for (uint32_t l = 0; l < L; l++)
        if (lane_node[l] == members[m]) {
          ms.lane_of_idx[m] = (uint8_t)l;
          ms.idx_of_lane[l] = (uint8_t)m;
          ms.lane_mask |= (uint16_t)(1u << l);
        }
    }
    for (uint32_t g = 0; g < G; g++) meta[g] = (R << 16) | (live && live[g] ? GPX_META_LIVE : 0u);
    memset(&S, 0, sizeof S);
    S.G = G;
    S.L = L;
    S.W = W;
    S.Rcap = Rcap;
    S.grp_meta = meta.data();
    S.msets = &ms;
    S.ctr = ctr.data();
    S.log_pos = log_pos.data();
    S.lp = 1; /* the copy of the ring heads the next launch would read */
  }
  /* lane's ring as the device holds it (ring_cap bytes, positions taken modulo ring_cap) up to head */
  void ring(uint32_t lane, uint8_t* ring, uint64_t ring_cap, uint64_t head) {
    S.ring[lane] = ring;
    S.ring_cap = ring_cap;
    log_pos[((size_t)S.lp * GPX_MAX_LANES + lane) * 2] = head;
  }
  StateEnv env() { return StateEnv{S, &ex.buf, &ex.bytes}; }
  /* what a wrapper returns: the kernel launches the call counted, or its GPX_* error code */
  int done(int rc) const { return rc ? rc : (int)ctr[C_KERNEL_LAUNCHES]; }
};
