/* gpx_state_seq.h -- the host sequence of every group-state and log-index call whose kernels are scalar:
 * gpx_log_find, gpx_log_gather, gpx_select_groups, gpx_missing_decisions, gpx_clear_group_flags, gpx_pause_groups and
 * gpx_handle_prepare_replies.  Each holds the argument checks, the scratch layout, the uploads, the settle, the launches
 * and the read-back, written once as a function template over an executor, as gpx_wire_seq.h does for the wire calls:
 * nvcc compiles it into the product (gpx_engine.cu: the CUDA executor) and g++ into the CPU tests (tests/emu: the CPU
 * executor).  Included by gpx_engine.cu after gpx_wire_seq.h.
 *
 * The executor is gpx_wire_seq.h's, plus
 *   ex.settle()    the lockstep records back into the group-state planes, before a kernel that reads or writes them
 * Its grow() keeps nothing across a reallocation: these layouts are laid out once per call.  A call object `call` has
 * begin(), which runs once the arguments pass and orders the log readers after the rounds issued on any stream. */
#pragma once

#include "gpx_logfind.cuh"
#include "gpx_pause.cuh"
#include "gpx_phase1b.cuh"
#include "gpx_wire_seq.h"

#include <vector>

/* what a sequence works on: the engine's state, read by reference, and its group-management scratch */
struct StateEnv {
  const DevState& S;
  void** buf;
  size_t* bytes;
};

/* some gid appears twice: two threads would read-modify-write the same group */
static bool gid_twice(std::vector<uint32_t> g) {
  std::sort(g.begin(), g.end());
  return std::adjacent_find(g.begin(), g.end()) != g.end();
}

/* ---- log index (gpx_logfind.cuh) ------------------------------------------------------------------------------------ */
/* gpx_log_find: k_log_dir -> k_log_scan over scan_threads threads -> k_log_hits.  The head is read on the device. */
template <class Ex, class C>
static int log_find(Ex& ex, C& call, const StateEnv& E, uint32_t lane, uint64_t from, uint32_t n,
                    const gpx_log_want* wants, gpx_log_hit* out, uint32_t scan_threads) {
  if (lane >= E.S.L) return fail(GPX_ERANGE, "lane");
  if (n == 0) return GPX_OK;
  if (!wants || !out) return fail(GPX_EINVAL, "null argument");
  if (from & 31) return fail(GPX_EINVAL, "from is not a segment boundary");
  for (uint32_t i = 0; i < n; i++) {
    if (wants[i].n_slots > GPX_LOG_SPAN) return fail(GPX_ERANGE, "n_slots > GPX_LOG_SPAN");
    if (i && wants[i - 1].gid >= wants[i].gid) return fail(GPX_EINVAL, "wants must be sorted by gid, one per group");
  }
  int rc = call.begin();
  if (rc) return rc;
  const size_t cells = (size_t)n * GPX_LOG_SPAN;
  LogFindArgs A;
  A.lane = lane;
  A.n = n;
  A.from = from;
  /* a segment is at least GPX_SEG_DEC_BYTES(1) = 96 bytes; a directory of 2^20 entries (32 MiB) covers every ring the
   * launches of this engine can fill with fewer segments than that, else LOGF_TOO_MANY */
  A.seg_cap = (uint32_t)std::min<uint64_t>(E.S.ring_cap / GPX_SEG_DEC_BYTES(1) + 2, 1ull << 20);
  gpx_log_want* d_wants;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
         d_wants = c.take<gpx_log_want>(n);
         A.segs = c.take<LogSeg>(A.seg_cap);
         A.ctl = c.take<unsigned long long>(4 + 2 * cells); /* [ctl | best], zeroed together */
         A.hits = c.take<gpx_log_hit>(cells);
         return (size_t)0;
       })))
    return rc;
  A.wants = d_wants;
  A.best = A.ctl + 4;
  unsigned long long ctl[4];
  if ((rc = ex.upload(d_wants, wants, (size_t)n * sizeof(gpx_log_want))) ||
      (rc = ex.fill(A.ctl, 0, (4 + 2 * cells) * 8)) || (rc = ex.launch(k_log_dir, 1, 32, E.S, A)) ||
      (rc = ex.launch(k_log_scan, scan_threads, GPX_LOGF_BLOCK, E.S, A)) ||
      (rc = ex.launch(k_log_hits, cells, GPX_LOGF_BLOCK, E.S, A)) || (rc = ex.read(ctl, A.ctl, sizeof ctl)) ||
      (rc = ex.read(out, A.hits, cells * sizeof(gpx_log_hit))) || (rc = ex.sync()))
    return rc;
  if (ctl[LOGF_ERR] == LOGF_OVERWRITTEN) return fail(GPX_ERANGE, "bytes from `from` on were already overwritten");
  if (ctl[LOGF_ERR] == LOGF_CORRUPT) return fail(GPX_EINVAL, "`from` is not a segment boundary");
  if (ctl[LOGF_ERR] == LOGF_TOO_MANY) return fail(GPX_ERANGE, "more log segments than the scan's directory holds");
  return GPX_OK;
}

/* gpx_log_gather: k_log_gather packs the ranges into the scratch for one copy.  call.begin() leaves the lane's head in
 * call.head. */
template <class Ex, class C>
static int log_gather(Ex& ex, C& call, const StateEnv& E, uint32_t lane, uint32_t n, const gpx_log_range* ranges,
                      void* dst, uint64_t dst_bytes) {
  if (lane >= E.S.L) return fail(GPX_ERANGE, "lane");
  if (n == 0) return GPX_OK;
  if (!ranges || !dst) return fail(GPX_EINVAL, "null argument");
  int rc = call.begin();
  if (rc) return rc;
  const uint64_t head = call.head, cap = E.S.ring_cap;
  std::vector<uint32_t> first(n + 1);
  uint64_t chunks = 0, top = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint64_t nc = ((uint64_t)ranges[i].len + 15) >> 4;
    if ((ranges[i].pos & 15) || (ranges[i].dst_off & 15)) return fail(GPX_EINVAL, "range not on a 16-byte boundary");
    if (ranges[i].pos + 16 * nc > head || head - ranges[i].pos > cap) return fail(GPX_ERANGE, "range outside the live ring bytes");
    if ((ranges[i].pos & (cap - 1)) + 16 * nc > cap) return fail(GPX_ERANGE, "range straddles the ring end");
    if ((uint64_t)ranges[i].dst_off + 16 * nc > dst_bytes) return fail(GPX_ERANGE, "range beyond dst");
    first[i] = (uint32_t)chunks;
    chunks += nc;
    top = std::max<uint64_t>(top, (uint64_t)ranges[i].dst_off + 16 * nc);
    if (chunks > 0xffffffffull) return fail(GPX_ERANGE, "too many bytes for one gather");
  }
  first[n] = (uint32_t)chunks;
  if (chunks == 0) return GPX_OK;
  LogGatherArgs A;
  A.lane = lane;
  A.n = n;
  gpx_log_range* d_ranges;
  uint32_t* d_first;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
         d_ranges = c.take<gpx_log_range>(n);
         d_first = c.take<uint32_t>(n + 1);
         A.out = c.take<int4>(top / 16);
         return (size_t)0;
       })))
    return rc;
  A.ranges = d_ranges;
  A.first_chunk = d_first;
  if ((rc = ex.upload(d_ranges, ranges, (size_t)n * sizeof(gpx_log_range))) ||
      (rc = ex.upload(d_first, first.data(), (size_t)(n + 1) * 4)) ||
      (rc = ex.fill(A.out, 0, top)) || /* gaps between ranges read as zero */
      (rc = ex.launch(k_log_gather, (uint32_t)chunks, GPX_LOGF_BLOCK, E.S, A)) || (rc = ex.read(dst, A.out, top)) ||
      (rc = ex.sync()))
    return rc;
  return GPX_OK;
}

/* ---- group sweeps (gpx_pause.cuh) ----------------------------------------------------------------------------------- */
/* gpx_select_groups: k_select_groups over every gid appends the matches in no fixed order; the host sorts them */
template <class Ex>
static int select_groups(Ex& ex, const StateEnv& E, uint32_t lane, uint32_t mask, uint32_t value, uint32_t* out_gids,
                         uint32_t cap, uint32_t* n_found) {
  if (!n_found || (!out_gids && cap)) return fail(GPX_EINVAL, "null argument");
  if (lane >= E.S.L) return fail(GPX_ERANGE, "lane");
  SelectArgs A;
  A.lane = lane;
  A.mask = mask;
  A.value = value;
  A.cap = cap;
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
    A.n_found = c.take<unsigned long long>(1);
    A.gids = c.take<uint32_t>(cap);
    return (size_t)0;
  });
  if (rc) return rc;
  unsigned long long found = 0;
  if ((rc = ex.fill(A.n_found, 0, 8)) || (rc = ex.settle()) ||
      (rc = ex.launch(k_select_groups, E.S.G, GPX_PAUSE_BLOCK, E.S, A)) || (rc = ex.read(&found, A.n_found, 8)) ||
      (rc = ex.sync()))
    return rc;
  const uint32_t got = (uint32_t)std::min<unsigned long long>(found, cap);
  if (got) {
    if ((rc = ex.read(out_gids, A.gids, (size_t)got * 4)) || (rc = ex.sync())) return rc;
    std::sort(out_gids, out_gids + got);
  }
  *n_found = (uint32_t)std::min<unsigned long long>(found, 0xffffffffull);
  return GPX_OK;
}

/* gpx_missing_decisions: one k_missing_decisions thread per gid */
template <class Ex>
static int missing_decisions(Ex& ex, const StateEnv& E, uint32_t lane, uint32_t n, const uint32_t* gids,
                             int32_t size_limit, int32_t too_much_gap, gpx_missing_rec* out) {
  if ((!gids || !out) && n) return fail(GPX_EINVAL, "null argument");
  if (lane >= E.S.L) return fail(GPX_ERANGE, "lane");
  if (n == 0) return GPX_OK;
  MissingArgs A;
  A.lane = lane;
  A.n = n;
  A.size_limit = size_limit;
  A.too_much_gap = too_much_gap;
  uint32_t* d_gids;
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
    d_gids = c.take<uint32_t>(n);
    A.out = c.take<gpx_missing_rec>(n);
    return (size_t)0;
  });
  if (rc) return rc;
  A.gids = d_gids;
  if ((rc = ex.upload(d_gids, gids, (size_t)n * 4)) || (rc = ex.settle()) ||
      (rc = ex.launch(k_missing_decisions, n, GPX_PAUSE_BLOCK, E.S, A)) ||
      (rc = ex.read(out, A.out, (size_t)n * sizeof(gpx_missing_rec))) || (rc = ex.sync()))
    return rc;
  return GPX_OK;
}

/* gpx_clear_group_flags: one k_clear_flags thread per gid */
template <class Ex>
static int clear_group_flags(Ex& ex, const StateEnv& E, uint32_t lane, uint32_t n, const uint32_t* gids, uint32_t mask) {
  if (!gids && n) return fail(GPX_EINVAL, "null argument");
  if (lane >= E.S.L) return fail(GPX_ERANGE, "lane");
  if (n == 0) return GPX_OK;
  if (gid_twice(std::vector<uint32_t>(gids, gids + n))) return fail(GPX_EINVAL, "a gid appears twice in the batch");
  uint32_t* d_gids;
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
    d_gids = c.take<uint32_t>(n);
    return (size_t)0;
  });
  if (rc || (rc = ex.upload(d_gids, gids, (size_t)n * 4)) || (rc = ex.settle()) ||
      (rc = ex.launch(k_clear_flags, n, 128, E.S, lane, (const uint32_t*)d_gids, n, mask)) || (rc = ex.sync()))
    return rc;
  return GPX_OK;
}

/* gpx_pause_groups up to the rows' host fields: one k_pause_groups thread per gid, then the rows of the paused groups,
 * the only ones the kernel writes, copied back as runs of consecutive paused entries */
template <class Ex>
static int pause_groups(Ex& ex, const StateEnv& E, uint32_t n, const uint32_t* gids, gpx_row* out_rows,
                        uint8_t* out_paused) {
  if (n == 0) return GPX_OK;
  if (!gids || !out_rows || !out_paused) return fail(GPX_EINVAL, "null argument");
  if (gid_twice(std::vector<uint32_t>(gids, gids + n))) return fail(GPX_EINVAL, "a gid appears twice in the batch");
  const uint32_t L = E.S.L;
  PauseArgs A;
  A.n = n;
  uint32_t* d_gids;
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
    d_gids = c.take<uint32_t>(n);
    A.rows = c.take<gpx_row>((size_t)n * L);
    A.paused = c.take<uint8_t>(n);
    return (size_t)0;
  });
  if (rc) return rc;
  A.gids = d_gids;
  if ((rc = ex.upload(d_gids, gids, (size_t)n * 4)) || (rc = ex.settle()) ||
      (rc = ex.launch(k_pause_groups, n, GPX_PAUSE_BLOCK, E.S, A)) || (rc = ex.read(out_paused, A.paused, n)) ||
      (rc = ex.sync()))
    return rc;
  for (uint32_t i = 0; i < n;) {
    if (!out_paused[i]) {
      i++;
      continue;
    }
    uint32_t j = i;
    while (j < n && out_paused[j]) j++;
    if ((rc = ex.read(out_rows + (size_t)i * L, A.rows + (size_t)i * L, (size_t)(j - i) * L * sizeof(gpx_row))))
      return rc;
    i = j;
  }
  return ex.sync();
}

/* ---- phase 1b (gpx_phase1b.cuh) ------------------------------------------------------------------------------------- */
/* gpx_handle_prepare_replies: one k_prepare_tally thread per election, over [elections | replies | out] */
template <class Ex>
static int prepare_replies(Ex& ex, const StateEnv& E, uint32_t n, const gpx_election_rec* elections,
                           uint32_t n_reply_recs, const gpx_prepare_reply_rec* replies, gpx_election_out* out) {
  if (n == 0) return GPX_OK;
  if (!elections || !out || (!replies && n_reply_recs)) return fail(GPX_EINVAL, "null argument");
  std::vector<uint32_t> gids(n);
  for (uint32_t i = 0; i < n; i++) {
    if ((uint64_t)elections[i].first_reply + elections[i].n_replies > n_reply_recs)
      return fail(GPX_ERANGE, "election refers to replies beyond n_reply_recs");
    gids[i] = elections[i].gid;
  }
  if (gid_twice(std::move(gids))) return fail(GPX_EINVAL, "more than one election for a group in one call");
  Phase1bArgs A;
  A.n = n;
  gpx_election_rec* d_els;
  gpx_prepare_reply_rec* d_replies;
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
    d_els = c.take<gpx_election_rec>(n);
    d_replies = c.take<gpx_prepare_reply_rec>(n_reply_recs);
    A.out = c.take<gpx_election_out>(n);
    return (size_t)0;
  });
  if (rc) return rc;
  A.els = d_els;
  A.replies = d_replies;
  if ((rc = ex.upload(d_els, elections, (size_t)n * sizeof(gpx_election_rec))) ||
      (n_reply_recs && (rc = ex.upload(d_replies, replies, (size_t)n_reply_recs * sizeof(gpx_prepare_reply_rec)))) ||
      (rc = ex.settle()) || (rc = ex.launch(k_prepare_tally, n, GPX_P1B_BLOCK, E.S, A)) ||
      (rc = ex.read(out, A.out, (size_t)n * sizeof(gpx_election_out))) || (rc = ex.sync()))
    return rc;
  return GPX_OK;
}
