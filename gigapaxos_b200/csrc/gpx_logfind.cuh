/*
 * gpx_logfind.cuh -- the journal's index as a scan of the log ring (the contract is the comment above gpx_log_find in
 * include/gpx.h): AbstractPaxosLogger.getLoggedDecisions :582 / getLoggedAccepts :568 in their journaling form,
 * SQLPaxosLogger.getLoggedFromMessageLog :3674-3756 over paxosutil/LogIndex.java:213-248, for a batch of
 * (group, slot range) wants.
 *
 *   k_log_dir   one thread walks the segment headers of one lane's ring from a known boundary to the head (a header
 *               names its own absolute position, so stale bytes of an earlier lap and the tail a launch skipped at
 *               the ring end are told from segments) and writes a directory {position, images, image size, type,
 *               index of its first image};
 *   k_log_scan  one thread per logged image (grid-stride over the directory's image count, which only the device
 *               knows): its group is looked up in the sorted wants, its slot in the want's range, and
 *               (segment, image) + 1 goes into the slot's cell with atomicMax -- the entry logged LAST wins, as
 *               `accepts.put(packet.slot, packet)` :3746 in log order;
 *   k_log_hits  one thread per wanted slot copies the winning DECISION and ACCEPT images (an ACCEPT image is two
 *               planes: 32-byte pvalue header, 16-byte {payload_off, payload_len, nreq, sender}) and the absolute
 *               position of the ACCEPT's request blob.
 *
 * Bytes: the scan reads 32 B per logged image once (a 1 GiB ring: ~0.2 ms at the HBM copy rate) instead of keeping a
 * per-group index up to date on the hot path.  Plain C++ over gpx_dev.cuh: tests/emu/ runs this source on the host.
 */
#pragma once
#include "gpx_dev.cuh"

struct LogSeg { /* 32 B */
  unsigned long long pos; /* absolute ring position of the segment header */
  uint32_t n_valid;       /* images in use */
  uint32_t n_slots;       /* images reserved */
  uint32_t rec_bytes;     /* 48: ACCEPT (two planes); 32: DECISION / PREPARE */
  uint32_t type;          /* GPX_F_ACCEPT | GPX_F_DECISION | GPX_F_PREPARE */
  uint32_t first_img;     /* index of its first image among all images of the directory */
  uint32_t pad;
};
enum { LOGF_NSEG = 0, LOGF_NIMG = 1, LOGF_ERR = 2, LOGF_HEAD = 3 }; /* words of the control block */
enum { LOGF_OK = 0, LOGF_OVERWRITTEN = 1, LOGF_CORRUPT = 2, LOGF_TOO_MANY = 3 };

struct LogFindArgs {
  uint32_t lane;
  uint32_t n; /* wants */
  unsigned long long from;
  const gpx_log_want* wants;
  LogSeg* segs;
  uint32_t seg_cap;
  unsigned long long* ctl;  /* [4] */
  unsigned long long* best; /* [2][n * GPX_LOG_SPAN]: 0 = none, else (segment << 32 | image) + 1; [0] DECISION, [1] ACCEPT */
  gpx_log_hit* hits;        /* [n * GPX_LOG_SPAN] */
};

__global__ void k_log_dir(const __grid_constant__ DevState S, const __grid_constant__ LogFindArgs A) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  atomicAdd(&S.ctr[C_KERNEL_LAUNCHES], 1ull);
  const unsigned long long cap = S.ring_cap;
  const unsigned long long head = S.log_pos[((size_t)S.lp * GPX_MAX_LANES + A.lane) * 2];
  unsigned long long pos = A.from, nimg = 0;
  uint32_t nseg = 0, err = LOGF_OK;
  if (head > pos && head - pos > cap) err = LOGF_OVERWRITTEN;
  while (err == LOGF_OK && pos + 64 <= head) {
    bool valid = (pos & (cap - 1)) + 64 <= cap; /* a header never straddles the ring end */
    gpx_log_seg_hdr h;
    if (valid) {
      h = *reinterpret_cast<const gpx_log_seg_hdr*>(ring_ptr(S, A.lane, pos));
      valid = h.magic == GPX_SEG_MAGIC && h.ring_off == pos;
    }
    if (!valid) { /* the tail a launch skipped (it would have straddled the ring end): on to the next lap */
      const unsigned long long nxt = (pos & ~(cap - 1)) + cap; /* the ring size is a power of two */
      if (nxt <= pos || nxt + 64 > head) break;
      pos = nxt;
      continue;
    }
    if ((h.rec_bytes != 32u && h.rec_bytes != 48u) || h.n_valid > h.n_slots) {
      err = LOGF_CORRUPT;
      break;
    }
    if (nseg == A.seg_cap || nimg + h.n_valid > 0xffffffffull) {
      err = LOGF_TOO_MANY;
      break;
    }
    LogSeg sg;
    sg.pos = pos;
    sg.n_valid = h.n_valid;
    sg.n_slots = h.n_slots;
    sg.rec_bytes = h.rec_bytes;
    sg.type = h.type;
    sg.first_img = (uint32_t)nimg;
    sg.pad = 0;
    A.segs[nseg++] = sg;
    nimg += h.n_valid;
    const unsigned long long body = (unsigned long long)h.n_slots * h.rec_bytes;
    if (body > cap || h.payload_bytes > cap) { /* sizes no launch of this engine writes: do not follow them */
      err = LOGF_CORRUPT;
      break;
    }
    const unsigned long long next = seg_end(pos, h);
    if (next - pos > cap) {
      err = LOGF_CORRUPT;
      break;
    }
    pos = next;
  }
  A.ctl[LOGF_NSEG] = nseg;
  A.ctl[LOGF_NIMG] = nimg;
  A.ctl[LOGF_ERR] = err;
  A.ctl[LOGF_HEAD] = head;
}

#define GPX_LOGF_BLOCK 256

__global__ void __launch_bounds__(GPX_LOGF_BLOCK) k_log_scan(const __grid_constant__ DevState S,
                                                             const __grid_constant__ LogFindArgs A) {
  if (A.ctl[LOGF_ERR] != LOGF_OK) return;
  const uint32_t nseg = (uint32_t)A.ctl[LOGF_NSEG];
  const unsigned long long nimg = A.ctl[LOGF_NIMG];
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  const size_t cells = (size_t)A.n * GPX_LOG_SPAN;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; idx < nimg; idx += stride) {
    uint32_t lo = 0, hi = nseg; /* the last segment whose first image is <= idx (empty segments share an index) */
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (A.segs[mid].first_img <= idx) lo = mid;
      else hi = mid;
    }
    const LogSeg sg = A.segs[lo];
    const uint32_t j = (uint32_t)(idx - sg.first_img);
    const bool isAcc = sg.rec_bytes == 48u, isDec = sg.rec_bytes == 32u && sg.type == GPX_F_DECISION;
    if (!isAcc && !isDec) continue; /* logged PREPAREs */
    const gpx_pvalue_hdr* img = reinterpret_cast<const gpx_pvalue_hdr*>(ring_ptr(S, A.lane, GPX_SEG_IMG(sg.pos, j)));
    const uint32_t gid = img->gid;
    if (img->flags & GPX_F_VOID) continue;
    uint32_t a = 0, b = A.n; /* the want of this group */
    while (a < b) {
      const uint32_t mid = (a + b) >> 1;
      if (A.wants[mid].gid < gid) a = mid + 1;
      else b = mid;
    }
    if (a >= A.n || A.wants[a].gid != gid) continue;
    const int k = jsub(img->slot, A.wants[a].min_slot);
    if (k < 0 || (uint32_t)k >= A.wants[a].n_slots || k >= GPX_LOG_SPAN) continue;
    atomicMax(&A.best[(isAcc ? cells : 0) + (size_t)a * GPX_LOG_SPAN + (uint32_t)k], (((unsigned long long)lo << 32) | j) + 1ull);
  }
}

__global__ void __launch_bounds__(GPX_LOGF_BLOCK) k_log_hits(const __grid_constant__ DevState S,
                                                             const __grid_constant__ LogFindArgs A) {
  const size_t cells = (size_t)A.n * GPX_LOG_SPAN;
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= cells) return;
  gpx_log_hit hit;
  memset(&hit, 0, sizeof hit);
  hit.decision.flags = GPX_F_VOID;
  hit.accept.h.flags = GPX_F_VOID;
  if (A.ctl[LOGF_ERR] == LOGF_OK) {
    const unsigned long long bd = A.best[t], ba = A.best[cells + t];
    if (bd) {
      const LogSeg sg = A.segs[(uint32_t)((bd - 1ull) >> 32)];
      const uint32_t j = (uint32_t)((bd - 1ull) & 0xffffffffull);
      hit.decision = *reinterpret_cast<const gpx_decision_rec*>(ring_ptr(S, A.lane, GPX_SEG_IMG(sg.pos, j)));
    }
    if (ba) {
      const LogSeg sg = A.segs[(uint32_t)((ba - 1ull) >> 32)];
      const uint32_t j = (uint32_t)((ba - 1ull) & 0xffffffffull);
      hit.accept.h = *reinterpret_cast<const gpx_pvalue_hdr*>(ring_ptr(S, A.lane, GPX_SEG_IMG(sg.pos, j)));
      const uint32_t* x = reinterpret_cast<const uint32_t*>(
          ring_ptr(S, A.lane, GPX_SEG_EXT(sg.pos, sg.n_slots, j)));
      hit.accept.payload_off = x[0];
      hit.accept.payload_len = x[1];
      hit.accept.nreq = x[2];
      hit.accept.sender = (int32_t)x[3];
      hit.blob_pos = sg.pos + GPX_SEG_PAY_OFF(sg.n_slots) + x[0];
    }
  }
  A.hits[t] = hit;
}

/* ---- k_log_gather: the request bodies of a batch of hits, packed for one device->host copy (gpx_log_gather) ------------
 * One thread per 16-byte chunk: chunk c belongs to the range r with first_chunk[r] <= c (binary search; the host lays the
 * ranges out back to back in chunks), is read from the ring at the range's position (blobs start on 16-byte boundaries
 * of a payload area padded to 16) and written to the staging buffer at the range's offset. */
struct LogGatherArgs {
  uint32_t lane, n;
  const gpx_log_range* ranges;
  const uint32_t* first_chunk; /* [n + 1] */
  int4* out;                   /* staging, indexed by dst_off / 16 */
};

__global__ void __launch_bounds__(GPX_LOGF_BLOCK) k_log_gather(const __grid_constant__ DevState S,
                                                               const __grid_constant__ LogGatherArgs A) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= A.first_chunk[A.n]) return;
  uint32_t lo = 0, hi = A.n; /* the last range whose first chunk is <= c (empty ranges share a chunk index) */
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (A.first_chunk[mid] <= c) lo = mid;
    else hi = mid;
  }
  const gpx_log_range r = A.ranges[lo];
  const uint32_t k = c - A.first_chunk[lo];
  A.out[(r.dst_off >> 4) + k] = *reinterpret_cast<const int4*>(ring_ptr(S, A.lane, r.pos + 16ull * k));
}
