/*
 * gpx_journal.cuh -- journal frames on the device (the contract is the comment above gpx_log_frame_device in
 * include/gpx.h): a range of one lane's log ring becomes the {int32 BE length}{packet} frames SQLPaxosLogger.journal
 * :965-1036 appends to its Journaler file, the bytes journal.LogDrainer writes for the same range.
 *
 *   k_log_dir          the segment directory of the range (gpx_logfind.cuh's walk, unchanged);
 *   k_journal_meta     one thread per table entry: the caller's (gid, req_id) table is strictly ascending;
 *   k_journal (emit 0) one thread per image (grid-stride over a host bound of the image count; the directory's count
 *                      is known on the device only): the name of its gid, a binary search of the table for its request
 *                      and every gpx_batch_ent of a batched blob, its frame's length, its misses;
 *   (exclusive scans of the three counter rows, then the one synchronisation for the totals and the flags)
 *   k_journal_fit      one thread per image: the frames' byte offsets stay within 32 bits;
 *   k_journal (emit 1) the misses at their scanned offsets, or (emit 2) the frames.
 *
 * The ACCEPT's RequestPacket bytes are gpx_wire_dev.cuh's ww_request_rec (the writer of gpx_wire_encode_accepts_device),
 * the JSON is gpx_wire_json_enc.cuh's writer (jw_head, jw_ballot, jw_i64), whose null buffer gives a length.  The
 * kernels read the ring, the name table and the caller's table, and no group-state plane.  Every kernel is scalar and
 * byte-addressed, so tests/emu compiles this file for the host.
 *
 * Bytes per image: the size pass reads its 32- (48-) byte image and the table's log2(n_meta) entries per request, the
 * emit pass the same again and the blob, and writes the frame: an ACCEPT of one request of v bytes is 94 + |paxosID|
 * + v bytes, a DECISION's JSON about 120 + |paxosID| bytes.
 */
#pragma once
#include "gpx_logfind.cuh"
#include "gpx_wire_json_enc.cuh"

/* words of the control block behind k_log_dir's (LOGF_*) */
enum { JF_UNSORTED = 4, JF_BAD_BLOB = 5, JF_OVER = 6, JF_NCTL = 8 };
/* counter rows per image: frame bytes, frames, misses */
enum { JF_BYTES = 0, JF_FRAMES = 1, JF_MISS = 2, JF_NCNT = 3 };

struct JournalArgs {
  uint32_t lane;
  uint32_t n;                   /* counter slots: a bound on the images of the range */
  const LogSeg* segs;           /* k_log_dir's directory */
  unsigned long long* ctl;      /* [JF_NCTL]: k_log_dir's LOGF_* words, then JF_* flags */
  const gpx_journal_req* meta;  /* [n_meta] ascending by (gid, req_id) */
  uint32_t n_meta;
  uint32_t* cnt;                /* [JF_NCNT][n] pass 0 */
  const uint32_t* off;          /* [JF_NCNT][n] their exclusive prefix sums */
  uint8_t* out;                 /* emit 2: the frames */
  gpx_journal_miss* miss;       /* emit 1: the misses */
  int emit;
};

__device__ __forceinline__ bool jf_less(const gpx_journal_req& a, uint32_t gid, int64_t req_id) {
  return a.gid < gid || (a.gid == gid && a.req_id < req_id);
}
/* the table's entry of (gid, req_id), or nullptr */
__device__ __forceinline__ const gpx_journal_req* jf_find(const JournalArgs& A, uint32_t gid, int64_t req_id) {
  uint32_t a = 0, b = A.n_meta;
  while (a < b) {
    const uint32_t mid = (a + b) >> 1;
    if (jf_less(A.meta[mid], gid, req_id)) a = mid + 1;
    else b = mid;
  }
  return a < A.n_meta && A.meta[a].gid == gid && A.meta[a].req_id == req_id ? &A.meta[a] : nullptr;
}

__global__ void k_journal_meta(const __grid_constant__ JournalArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 || i >= A.n_meta) return;
  const gpx_journal_req p = A.meta[i - 1], q = A.meta[i];
  if (!jf_less(p, q.gid, q.req_id)) A.ctl[JF_UNSORTED] = 1;
}

/* RequestPacket bytes of one logged request (ww_request_rec, gpx_wire_encode_accepts_device's writer): the fields the
 * ring holds, the table's entryReplica and entryTime, wire.Request's defaults for the rest */
__device__ __forceinline__ uint32_t jf_request(uint8_t* p, int32_t type, const WireNames& W, uint32_t gid, int64_t req_id,
                                               bool stop, const gpx_journal_req* r, const uint8_t* val, uint32_t len,
                                               uint32_t n_batched) {
  gpx_request_rec rq;
  memset(&rq, 0, sizeof rq);
  rq.gid = gid;
  rq.flags = stop ? GPX_F_STOP : 0u;
  rq.req_id = req_id;
  rq.payload_len = len;
  rq.entry_node = r->entry_node;
  gpx_wire_req_meta m;
  memset(&m, 0, sizeof m);
  m.entry_time = r->entry_time;
  return ww_request_rec(p, type, W, gid, rq, m, val, n_batched);
}

/* one image: its frame's bytes, written at o + 4 behind the length word unless o is null, and its misses, each passed
 * to miss(req_id) (-1: the gid has no name).  An image with a miss gets no frame (0 bytes); so does a VOID one. */
template <typename Miss>
__device__ __forceinline__ uint32_t jf_frame(const DevState& S, const WireNames& W, const JournalArgs& A, const LogSeg& sg,
                                             uint32_t j, uint8_t* o, uint32_t& kind, Miss miss) {
  const gpx_pvalue_hdr h = *reinterpret_cast<const gpx_pvalue_hdr*>(ring_ptr(S, A.lane, GPX_SEG_IMG(sg.pos, j)));
  const bool acc = sg.rec_bytes == 48u;
  kind = acc ? GPX_F_ACCEPT : (h.flags & GPX_F_PREPARE) ? GPX_F_PREPARE : GPX_F_DECISION;
  if (h.flags & GPX_F_VOID) return 0;
  if (W.slot == nullptr || h.gid >= S.G || W.slot[h.gid] == GPX_NAME_NONE) {
    miss(-1ll);
    return 0;
  }
  const uint32_t gid = h.gid;
  uint32_t b = 0;
  if (!acc) {
    const gpx_journal_req* r = kind == GPX_F_DECISION ? jf_find(A, gid, h.req_id) : nullptr;
    if (kind == GPX_F_DECISION && !r) {
      miss(h.req_id);
      return 0;
    }
    JsonW w{o ? o + 4 : nullptr, 0};
    if (kind == GPX_F_PREPARE) { /* journal.prepare_json: the slot field carries firstUndecidedSlot */
      jw_head(w, W, 2, gid);
      jw_ballot(w, h.bnum, h.bcoord);
      jw_s(w, ",\"PREP_MIN\":");
      jw_i64(w, h.slot);
    } else { /* journal.decision_json */
      jw_head(w, W, 6, gid);
      jw_ballot(w, h.bnum, h.bcoord);
      jw_s(w, ",\"GC_S\":");
      jw_i64(w, h.median_cp);
      jw_s(w, ",\"S\":");
      jw_i64(w, h.slot);
      jw_s(w, ",\"QID\":");
      jw_i64(w, h.req_id);
      jw_s(w, ",\"ET\":");
      jw_i64(w, r->entry_time);
      jw_s(w, ",\"E\":");
      jw_i64(w, r->entry_node);
      if (h.flags & GPX_F_STOP) jw_s(w, ",\"STOP\":true");
    }
    jw_c(w, '}');
    b = w.n;
  } else { /* AcceptPacket.toBytes :95-138 of wire.encode_accept */
    const uint32_t* x = reinterpret_cast<const uint32_t*>(ring_ptr(S, A.lane, GPX_SEG_EXT(sg.pos, sg.n_slots, j)));
    const uint32_t poff = x[0], plen = x[1], nreq = x[2];
    const int32_t sender = (int32_t)x[3];
    const uint8_t* blob = ring_ptr(S, A.lane, sg.pos + GPX_SEG_PAY_OFF(sg.n_slots) + poff);
    const gpx_batch_ent* ents = reinterpret_cast<const gpx_batch_ent*>(blob);
    const gpx_journal_req* r = jf_find(A, gid, h.req_id);
    bool whole = r != nullptr;
    if (!r) miss(h.req_id);
    if (nreq > 1)
      for (uint32_t k = 1; k < nreq; k++)
        if (!jf_find(A, gid, ents[k].req_id)) {
          miss(ents[k].req_id);
          whole = false;
        }
    if (!whole) return 0;
    uint8_t* p = o ? o + 4 : nullptr;
    if (nreq <= 1) {
      b = ww_request_bytes(W, gid, plen);
      if (p) b = jf_request(p, GPX_PT_ACCEPT, W, gid, h.req_id, (h.flags & GPX_F_STOP) != 0, r, blob, plen, 0);
    } else {
      const uint8_t* val = blob + 16u * nreq;
      b = ww_request_bytes(W, gid, ents[0].len);
      if (p) b = jf_request(p, GPX_PT_ACCEPT, W, gid, ents[0].req_id, (ents[0].flags & GPX_F_STOP) != 0, r, val,
                            ents[0].len, nreq - 1);
      val += ents[0].len;
      for (uint32_t k = 1; k < nreq; k++) {
        const gpx_batch_ent e = ents[k];
        uint32_t l = ww_request_bytes(W, gid, e.len);
        if (p) {
          const gpx_journal_req* s = jf_find(A, gid, e.req_id);
          l = jf_request(p + b + 4, GPX_PT_REQUEST, W, gid, e.req_id, (e.flags & GPX_F_STOP) != 0, s, val, e.len, 0);
          ww_i32(p + b, (int32_t)l);
        }
        b += 4u + l;
        val += e.len;
      }
    }
    if (p) {
      ww_i32(p + b, h.slot);
      ww_i32(p + b + 4, h.bnum);
      ww_i32(p + b + 8, h.bcoord);
      p[b + 12] = 0; /* recovery */
      ww_i32(p + b + 13, h.median_cp);
      p[b + 17] = 0; /* noCoalesce */
      ww_i32(p + b + 18, sender);
    }
    b += 22;
  }
  if (o) ww_i32(o, (int32_t)b);
  return 4u + b;
}

/* an ACCEPT image's blob lies inside its segment's payload area, and a batched one's entries and values inside the
 * blob: what k_log_dir's walk cannot vouch for, checked before any frame reads it */
__device__ __forceinline__ bool jf_blob_ok(const DevState& S, const JournalArgs& A, const LogSeg& sg, uint32_t j) {
  const gpx_log_seg_hdr* sh = reinterpret_cast<const gpx_log_seg_hdr*>(ring_ptr(S, A.lane, sg.pos));
  const uint32_t* x = reinterpret_cast<const uint32_t*>(ring_ptr(S, A.lane, GPX_SEG_EXT(sg.pos, sg.n_slots, j)));
  const uint64_t poff = x[0], plen = x[1], nreq = x[2];
  if (poff + plen > sh->payload_bytes) return false;
  if (nreq <= 1) return true;
  if ((poff & 15u) || 16u * nreq > plen) return false;
  const gpx_batch_ent* ents = reinterpret_cast<const gpx_batch_ent*>(ring_ptr(S, A.lane, sg.pos + GPX_SEG_PAY_OFF(sg.n_slots) + poff));
  uint64_t v = 16u * nreq;
  for (uint32_t k = 0; k < nreq; k++) v += ents[k].len;
  return v <= plen;
}

#define GPX_JOURNAL_BLOCK 128

__global__ void __launch_bounds__(GPX_JOURNAL_BLOCK) k_journal(const __grid_constant__ DevState S,
                                                               const __grid_constant__ WireNames W,
                                                               const __grid_constant__ JournalArgs A) {
  if (A.ctl[LOGF_ERR] != LOGF_OK) return;
  const uint32_t nseg = (uint32_t)A.ctl[LOGF_NSEG];
  const unsigned long long nimg = A.ctl[LOGF_NIMG];
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; idx < A.n; idx += stride) {
    if (idx >= nimg) { /* past the directory's images: empty counters */
      if (A.emit == 0)
        for (int r = 0; r < JF_NCNT; r++) A.cnt[(size_t)r * A.n + idx] = 0;
      continue;
    }
    uint32_t lo = 0, hi = nseg; /* the last segment whose first image is <= idx (empty segments share an index) */
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (A.segs[mid].first_img <= idx) lo = mid;
      else hi = mid;
    }
    const LogSeg sg = A.segs[lo];
    const uint32_t j = (uint32_t)(idx - sg.first_img);
    const gpx_pvalue_hdr* img = reinterpret_cast<const gpx_pvalue_hdr*>(ring_ptr(S, A.lane, GPX_SEG_IMG(sg.pos, j)));
    uint32_t kind;
    if (A.emit == 0) {
      uint32_t nm = 0;
      uint32_t bytes = 0;
      if (sg.rec_bytes == 48u && !(img->flags & GPX_F_VOID) && !jf_blob_ok(S, A, sg, j)) A.ctl[JF_BAD_BLOB] = 1;
      else bytes = jf_frame(S, W, A, sg, j, nullptr, kind, [&](int64_t) { nm++; });
      A.cnt[(size_t)JF_BYTES * A.n + idx] = nm ? 0u : bytes;
      A.cnt[(size_t)JF_FRAMES * A.n + idx] = !nm && bytes ? 1u : 0u;
      A.cnt[(size_t)JF_MISS * A.n + idx] = nm;
    } else if (A.emit == 1) {
      if (A.cnt[(size_t)JF_MISS * A.n + idx] == 0) continue;
      gpx_journal_miss* m = A.miss + A.off[(size_t)JF_MISS * A.n + idx];
      const uint32_t gid = img->gid;
      jf_frame(S, W, A, sg, j, nullptr, kind, [&](int64_t req_id) {
        gpx_journal_miss x;
        x.gid = gid;
        x.kind = kind;
        x.req_id = req_id;
        *m++ = x;
      });
    } else if (A.cnt[(size_t)JF_FRAMES * A.n + idx]) {
      jf_frame(S, W, A, sg, j, A.out + A.off[(size_t)JF_BYTES * A.n + idx], kind, [](int64_t) {});
    }
  }
}

/* the frames' offsets are 32-bit: flag a range whose frames pass 4 GiB (the scan wraps at the first such image) */
__global__ void k_journal_fit(const __grid_constant__ JournalArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < A.n && (unsigned long long)A.off[(size_t)JF_BYTES * A.n + i] + A.cnt[(size_t)JF_BYTES * A.n + i] > 0xffffffffull)
    A.ctl[JF_OVER] = 1;
}
