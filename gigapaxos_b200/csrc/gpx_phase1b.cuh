/*
 * gpx_phase1b.cuh -- k_prepare_tally: phase 1b at the would-be coordinators (PISM.handlePrepareReply :1017-1068,
 * PaxosCoordinator.getPreActivesIfPreempted PaxosCoordinator.java:313-318 / handlePrepareReply :281-299,
 * PaxosCoordinatorState.java:264-587; the contract is the comment above gpx_handle_prepare_replies in include/gpx.h).
 *
 * One thread per election (= one pre-active coordinator of one group).  The thread walks its PREPARE_REPLY records in
 * order -- a higher ballot preempts, lower ballots / strangers / repeats are ignored, recordSlotNumber takes
 * PrepareReplyPacket.getMinSlot(), the pvalue of the highest ballot per slot is carried over -- until a majority of
 * the members has been heard; then it lays out the plan (carried-over pvalue or no-op for every slot from the largest
 * recorded minimum to the largest carried-over slot, a fresh STOP behind a carried-over STOP that is not last), resigns
 * the local coordinators of a lower ballot and installs the new one ACTIVE with the recorded nodeSlotNumbers: the
 * writes GPX_PATCH_RESIGN_COORD / INSTALL_COORD / SET_NODE_SLOT would make, without the round trips.
 *
 * A mass fail-over (a node is lost: every group it coordinated elects at once) is one launch over all of them; per
 * election the work is a few hundred bytes of replies and a 896-byte result, so the kernel is written for clarity:
 * carry-over table (<= GPX_MAX_CARRY slots) and plan (<= GPX_MAX_PLAN + 1) live in local memory, searches are linear.
 * No warp-level primitives, no shared memory, no inline PTX: besides gpx_dev.cuh's index helpers this file is plain
 * C++, and tests/emu/ compiles it for the host to run the very same code against the oracle without a GPU.
 */
#pragma once
#include "gpx_dev.cuh"

struct Phase1bArgs {
  const gpx_election_rec* els;
  uint32_t n;
  const gpx_prepare_reply_rec* replies;
  gpx_election_out* out;
};

#define GPX_P1B_BLOCK 64

__global__ void __launch_bounds__(GPX_P1B_BLOCK) k_prepare_tally(const __grid_constant__ DevState S,
                                                                  const __grid_constant__ Phase1bArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) atomicAdd(&S.ctr[C_KERNEL_LAUNCHES], 1ull);
  if (i >= A.n) return;
  const gpx_election_rec el = A.els[i];
  gpx_election_out* o = &A.out[i];
  {
    int4* oz = reinterpret_cast<int4*>(o);
    for (uint32_t k = 0; k < (uint32_t)(sizeof(gpx_election_out) / 16); k++) oz[k] = make_int4(0, 0, 0, 0);
  }
  int ns[GPX_MAX_GROUP_SIZE]; /* nodeSlotNumbers, PCS ctor :169-171 */
  for (int m = 0; m < GPX_MAX_GROUP_SIZE; m++) ns[m] = -1;
  int verdict = GPX_EL_DROPPED;

  const uint32_t gid = el.gid;
  const GroupCtx g = group_ctx(S, gid);
  bool ok = g.live && el.lane < S.L;
  if (ok) ok = st_usable(S.acc_aux[row_idx(S, el.lane, gid)]) && g.ms->idx_of_lane[el.lane] != 0xffu; /* PISM :456-460 */

  if (ok) {
    const uint32_t R = g.R;
    const int bn = el.bnum, bc = el.bcoord;
    int c_slot[GPX_MAX_CARRY];                 /* carryoverProposals: slot -> (pvalue, record that carried it) */
    gpx_accepted_pvalue c_pv[GPX_MAX_CARRY];
    uint32_t c_src[GPX_MAX_CARRY];
    uint32_t ncarry = 0, heard = 0, nheard = 0;
    verdict = GPX_EL_WAITING;
    const uint32_t end = el.first_reply + el.n_replies;
    uint32_t k = el.first_reply;
    while (k < end && verdict == GPX_EL_WAITING) {
      /* one PREPARE_REPLY = the record at k and its GPX_F_MORE continuations [k, kend) */
      const gpx_prepare_reply_rec* h = &A.replies[k];
      const uint32_t who = h->who;
      const uint32_t idx = GPX_WHO_ACC(who), hfl = GPX_WHO_FLAGS(who);
      const int firstSlot = (int)((unsigned)h->first_slot + 1u); /* the record holds gcSlot; firstSlot = gcSlot + 1 */
      const int c = bcmp(h->bnum, h->bcoord, bn, bc);
      uint32_t kend = k + 1;
      for (uint32_t f = hfl; (f & GPX_F_MORE) && !(f & GPX_F_VOID) && kend < end; kend++) f = GPX_WHO_FLAGS(A.replies[kend].who);
      bool skip = (hfl & GPX_F_VOID) != 0;
      if (!skip && c > 0) { /* isPreemptable :271-278: the election is lost */
        verdict = GPX_EL_PREEMPTED;
        break;
      }
      if (!skip && (idx >= R || c < 0 || ((heard >> idx) & 1u))) skip = true; /* canIgnorePrepareReply :287-316 */
      if (!skip) {
        /* recordSlotNumber :786-807 with PrepareReplyPacket.getMinSlot() :151-164 */
        int minSlot = firstSlot;
        for (uint32_t kk = k; kk < kend; kk++) {
          const gpx_prepare_reply_rec* r = &A.replies[kk];
          const uint32_t na = r->n_accepted < (uint32_t)GPX_MAX_WINDOW ? r->n_accepted : (uint32_t)GPX_MAX_WINDOW;
          for (uint32_t a = 0; a < na; a++)
            if (jsub(r->accepted[a].slot, minSlot) < 0) minSlot = r->accepted[a].slot;
        }
        if (jsub(ns[idx], minSlot) < 0) ns[idx] = minSlot;
        /* isPrepareAcceptedByMajority :347-366: per slot the pvalue of the highest ballot */
        bool overflow = false;
        for (uint32_t kk = k; kk < kend && !overflow; kk++) {
          const gpx_prepare_reply_rec* r = &A.replies[kk];
          const uint32_t na = r->n_accepted < (uint32_t)GPX_MAX_WINDOW ? r->n_accepted : (uint32_t)GPX_MAX_WINDOW;
          for (uint32_t a = 0; a < na; a++) {
            const gpx_accepted_pvalue pv = r->accepted[a];
            uint32_t j = 0;
            while (j < ncarry && c_slot[j] != pv.slot) j++;
            if (j < ncarry) {
              if (bcmp(pv.bnum, pv.bcoord, c_pv[j].bnum, c_pv[j].bcoord) > 0) {
                c_pv[j] = pv;
                c_src[j] = kk;
              }
            } else if (ncarry == (uint32_t)GPX_MAX_CARRY) { /* device rule */
              overflow = true;
              break;
            } else {
              c_slot[ncarry] = pv.slot;
              c_pv[ncarry] = pv;
              c_src[ncarry] = kk;
              ncarry++;
            }
          }
        }
        if (overflow) {
          verdict = GPX_EL_OVERFLOW;
        } else {
          heard |= 1u << idx; /* waitforMyBallot.updateHeardFrom */
          nheard++;
          if (nheard > R / 2) verdict = GPX_EL_MAJORITY; /* WaitforUtility.heardFromMajority :64-68 */
        }
      }
      k = kend;
    }

    if (verdict == GPX_EL_MAJORITY) {
      /* combinePValuesOntoProposals :393-444 (no pre-active proposals: see include/gpx.h) */
      int p_slot[GPX_MAX_PLAN + 1];
      uint32_t p_kind[GPX_MAX_PLAN + 1];
      bool p_stop[GPX_MAX_PLAN + 1];
      uint32_t np = 0, flags = 0;
      int nextSlot = el.slot; /* PCS ctor: nextProposalSlotNumber = paxosState.getSlot() */
      if (ncarry > 0) {
        int maxCarry = c_slot[0]; /* getMaxPValueSlot :903-914 */
        for (uint32_t j = 1; j < ncarry; j++)
          if (jsub(c_slot[j], maxCarry) > 0) maxCarry = c_slot[j];
        int maxMin = ns[0]; /* getMaxMinCarryoverSlot :921-931 */
        for (uint32_t m = 1; m < R; m++)
          if (jsub(ns[m], maxMin) > 0) maxMin = ns[m];
        const int span = jsub(maxCarry, maxMin); /* slots to fill - 1; negative: every carried-over slot lies below maxMin */
        if (span >= GPX_MAX_PLAN) {
          verdict = GPX_EL_OVERFLOW; /* device rule */
        } else {
          /* for (curSlot = maxMin; curSlot - maxCarry <= 0; curSlot++) :408, counted so that no pair of slots (not even
           * two that are 2^31 apart in a hostile record) can make it run away */
          for (int d = 0; d <= span; d++) {
            const int cur = (int)((unsigned)maxMin + (unsigned)d);
            uint32_t j = 0;
            while (j < ncarry && c_slot[j] != cur) j++;
            gpx_carryover* e = &o->plan[np];
            e->slot = cur;
            if (j < ncarry) {
              e->kind = GPX_CO_PVALUE;
              e->src_reply = c_src[j];
              e->pv = c_pv[j];
              p_stop[np] = (c_pv[j].flags & 2u) != 0;
            } else {
              e->kind = GPX_CO_NOOP; /* makeNoopPValue :886-897 */
              p_stop[np] = false;
            }
            p_slot[np] = cur;
            p_kind[np] = e->kind;
            np++;
          }
          nextSlot = (int)((unsigned)maxCarry + 1u); /* :436 */
          /* processStop :478-554: all ballots are the new one here, nothing is converted; a regular request behind a
           * STOP is the reference's assert(false) :524 */
          bool stopExists = false;
          for (uint32_t a = 0; a < np; a++) {
            if (!p_stop[a]) continue;
            stopExists = true;
            for (uint32_t b = 0; b < np; b++)
              if (!p_stop[b] && p_kind[b] != GPX_CO_NOOP && jsub(p_slot[a], p_slot[b]) < 0) flags |= GPX_ELF_STOP_ORDER;
          }
          if (stopExists && np > 0 && !p_stop[np - 1]) { /* :538-542: propose(new RequestPacket(0, STOP, true)) */
            gpx_carryover* e = &o->plan[np];
            e->slot = nextSlot;
            e->kind = GPX_CO_STOP_NEW;
            p_slot[np] = nextSlot;
            np++;
            nextSlot = (int)((unsigned)nextSlot + 1u);
          }
        }
      }
      if (verdict == GPX_EL_MAJORITY) {
        const int installed = np > 0 ? p_slot[0] : nextSlot;
        o->next_slot = installed;
        o->n_plan = (uint16_t)np;
        o->flags = (uint16_t)flags;
        /* coordinators of a lower ballot resign (what GPX_PATCH_RESIGN_COORD writes) ... */
        for (uint32_t l = 0; l < S.L; l++) {
          const size_t ri = row_idx(S, l, gid);
          const int4 cr = S.coord_row[ri];
          if (l != el.lane && ((unsigned)cr.w & GPX_CF_EXISTS) && bcmp(cr.x, cr.y, bn, bc) > 0) continue;
          S.coord_row[ri] = make_int4(0, 0, 0, 0);
          for (uint32_t w = 0; w < S.W; w++) S.prop_win[win_idx(S, l, w, gid)] = make_int4(0, 0, 0, 0);
        }
        /* ... and the new one starts ACTIVE at the plan's first slot (GPX_PATCH_INSTALL_COORD + SET_NODE_SLOT x R;
         * setCoordinatorActive :577-587) */
        S.coord_row[row_idx(S, el.lane, gid)] = make_int4(bn, bc, installed, (int)(GPX_CF_EXISTS | GPX_CF_ACTIVE));
        int nv[GPX_MAX_GROUP_SIZE];
        for (uint32_t m = 0; m < S.Rcap; m++) nv[m] = m < R && jsub(-1, ns[m]) < 0 ? ns[m] : -1;
        ns_put(S, el.lane, gid, R, S.Rcap, nv);
      }
    }
  }
  o->gid = gid;
  o->verdict = verdict;
  for (int m = 0; m < GPX_MAX_GROUP_SIZE; m++) o->node_slots[m] = ns[m];
}
