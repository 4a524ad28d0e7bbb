/*
 * gpx_journal_gc.cuh -- journal garbage collection on the device (the contract is the comment above
 * gpx_journal_compact_device in include/gpx.h): the frames of k journal files that a checkpoint still needs, in the
 * files' byte format, as SQLPaxosLogger.compactLogfile :3350-3450 rewrites each file to what LogIndex.isLogMsgNeeded
 * :331-345 wants.  journal.compact_files is the host model these kernels are tested against.
 *
 *   k_jgc_offsets  one thread per file boundary: file_off is ascending from 0 to n_bytes;
 *   k_jgc_parse    one thread per frame: its length agrees with the next start and stays in its file; the packet
 *                  parses as an ACCEPT (gpx_wire_dev.cuh's reader), a DECISION or a PREPARE (gpx_wire_json.cuh's field
 *                  reader); its (paxosID, version) resolves through the name table as the wire decoders resolve it
 *                  (wire_name_find / json_id_gid, wire_group); the frame's sort key is its gid when it is indexed
 *                  (resolved, slot above the group's gc slot), else the count of groups;
 *   (the wire calls' stable sort by gid: a group's indexed frames are one run)
 *   k_jgc_keep     one thread per frame: the keep rule, a PREPARE scanning its group's run entry by entry;
 *   (exclusive scans of the frame counters)
 *   k_jgc_file     one thread per file: its frame range, counts, status and compacted bytes;
 *   (an exclusive scan of the compacted bytes over the files, then the one synchronisation)
 *   k_jgc_bad      the malformed frames' indices at their scanned offsets, or
 *   k_jgc_copy     one warp per kept frame of a compacted file: the frame copied unchanged, 4-byte stores aligned to
 *                  the destination; k_jgc_files the per-file records.
 *
 * The kernels read the frames, the name table, the group meta words (liveness) and the caller's gc slots, and no
 * group-state plane.  Every kernel is scalar (the copy's warp is 32 threads indexed from the global thread index, no
 * warp primitive), so tests/emu compiles this file for the host.
 *
 * Bytes per frame: the parse pass reads the frame (an ACCEPT's header and request fields, a JSON frame in full) and
 * the gc slot of its gid; the keep pass a 24-byte record (and a PREPARE its group's run); the copy reads and writes the
 * kept frames once.
 */
#pragma once
#include "gpx_wire_dev.cuh"
#include "gpx_wire_json.cuh"

/* counter rows per frame: kept frame bytes, kept frames, unresolved frames, malformed frames */
enum { JG_KBYTES = 0, JG_KEPT = 1, JG_UNRES = 2, JG_BAD = 3, JG_NCNT = 4 };
/* JgcRec.flags */
enum { JG_PREPARE = 1u, JG_RESOLVED = 2u, JG_INDEXED = 4u };
#define GPX_JGC_PT_PREPARE 2 /* PaxosPacketType.PREPARE */

struct JgcRec { /* one parsed frame */
  uint32_t len;   /* the packet's bytes (the frame is 4 + len) */
  uint32_t gid;   /* resolved frames */
  int32_t slot;   /* an ACCEPT's or DECISION's slot, a PREPARE's firstUndecidedSlot */
  int32_t bnum, bcoord;
  uint32_t flags;
};
struct JgcFile { /* one file before the outputs are written */
  gpx_journal_file f;
  uint32_t lo;    /* its first frame */
  uint32_t kb_lo; /* the kept-bytes scan at lo */
};

struct JournalGcArgs {
  const uint8_t* bytes;
  uint32_t n_bytes;
  const uint32_t* file_off; /* [n_files + 1] */
  uint32_t n_files;
  const uint32_t* starts;   /* [n] */
  uint32_t n;
  const int32_t* gc_slot;   /* [G] */
  uint32_t last_readonly;
  uint32_t* bad_off;        /* 1 word: file_off is not ascending from 0 to n_bytes */
  JgcRec* rec;              /* [n] */
  uint32_t* key;            /* [n] */
  uint32_t* cnt;            /* [JG_NCNT][n] */
  const uint32_t* off;      /* [JG_NCNT][n] their exclusive prefix sums */
  const uint32_t* tot;      /* [JG_NCNT] their totals */
  const uint32_t* perm;     /* the gid sort: frame of each sorted key */
  const uint32_t* skey;     /* the sorted keys */
  JgcFile* fs;              /* [n_files] */
  uint32_t* fbytes;         /* [n_files] compacted bytes */
  const uint32_t* foff;     /* [n_files] their exclusive prefix sums */
  uint8_t* out;
  gpx_journal_file* files;
  uint32_t* bad;
};

/* the file frame start s lies in: the last f < n_files with file_off[f] <= s (an empty file holds no frame) */
__device__ __forceinline__ uint32_t jg_file(const JournalGcArgs& A, uint32_t s) {
  uint32_t lo = 0, hi = A.n_files;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (A.file_off[mid] <= s) lo = mid;
    else hi = mid;
  }
  return lo;
}
/* the first frame whose start is >= x */
__device__ __forceinline__ uint32_t jg_first(const JournalGcArgs& A, uint32_t x) {
  uint32_t lo = 0, hi = A.n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (A.starts[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ uint32_t jg_be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}

/* the keys of a journaled DECISION (journal.decision_json) and PREPARE (journal.prepare_json), up to 8 ISO-8859-1
 * characters packed little-endian */
enum { JG_K_TYPE, JG_K_PT, JG_K_ID, JG_K_V, JG_K_B, JG_K_S, JG_K_GC_S, JG_K_QID, JG_K_ET, JG_K_E, JG_K_PREP, JG_K_N };
struct JgcKeys {
  enum { N = JG_K_N, PP = -2 }; /* no array to jump over */
  __device__ __forceinline__ static int id(const JStr& s, const JRd&, uint32_t) {
    if (s.wide) return -1;
    switch (s.len) {
      case 1:
        if (s.head == 'V') return JG_K_V;
        if (s.head == 'B') return JG_K_B;
        if (s.head == 'S') return JG_K_S;
        if (s.head == 'E') return JG_K_E;
        return -1;
      case 2:
        if (s.head == JK('P', 'T', 0, 0, 0)) return JG_K_PT;
        if (s.head == JK('I', 'D', 0, 0, 0)) return JG_K_ID;
        if (s.head == JK('E', 'T', 0, 0, 0)) return JG_K_ET;
        return -1;
      case 3: return s.head == JK('Q', 'I', 'D', 0, 0) ? JG_K_QID : -1;
      case 4:
        if (s.head == JK('t', 'y', 'p', 'e', 0)) return JG_K_TYPE;
        if (s.head == JK('G', 'C', '_', 'S', 0)) return JG_K_GC_S;
        return -1;
      case 8: return s.head == JK8('P', 'R', 'E', 'P', '_', 'M', 'I', 'N') ? JG_K_PREP : -1;
      default: return -1;
    }
  }
};
/* a required int64 at pos */
__device__ __forceinline__ bool jg_get_i64(const JRd& J0, uint32_t at, int64_t* v) {
  JRd J = J0;
  if (!json_at(J, at)) return false;
  *v = jr_i64(J);
  return J.ok;
}

/* the packet at bytes[at, at + len) as journal.parse_packet reads it: false when it is not an ACCEPT, a DECISION or a
 * PREPARE; else its slot, ballot and kind in x, its gid (GPX_NAME_NONE unless it resolves) in gid */
__device__ __forceinline__ bool jg_packet(const DevState& S, const WireNames& W, const JournalGcArgs& A, uint32_t at,
                                          uint32_t len, JgcRec& x, uint32_t& gid) {
  gid = GPX_NAME_NONE;
  int32_t version = 0;
  if (len > 0 && A.bytes[at] == '{') { /* DECISION / PREPARE JSON */
    JRd J;
    J.b = A.bytes;
    J.n = at;
    J.end = at + len;
    J.ok = true;
    uint32_t pos[JG_K_N], ppc = GPX_JSON_NONE;
    json_keys_t<JgcKeys>(J, pos, nullptr, &ppc);
    jr_ws(J);
    if (!J.ok || J.n != J.end) return false;
    int32_t type = 0, pt = 0, i32 = 0;
    int64_t i64 = 0;
    if (!json_get_i32(J, pos[JG_K_TYPE], &type) || type != GPX_PT_PAXOS_PACKET || !json_get_i32(J, pos[JG_K_PT], &pt))
      return false;
    if (!json_get_i32(J, pos[JG_K_V], &version) || !json_get_ballot(J, pos[JG_K_B], &x.bnum, &x.bcoord)) return false;
    if (!pos[JG_K_ID] || J.b[pos[JG_K_ID]] != '"') return false;
    if (pt == GPX_PT_DECISION) {
      if (!json_get_i32(J, pos[JG_K_S], &x.slot) || !json_get_i32(J, pos[JG_K_GC_S], &i32) ||
          !json_get_i32(J, pos[JG_K_E], &i32) || !jg_get_i64(J, pos[JG_K_QID], &i64) || !jg_get_i64(J, pos[JG_K_ET], &i64))
        return false;
      x.flags = 0;
    } else if (pt == GPX_JGC_PT_PREPARE) {
      if (!json_get_i32(J, pos[JG_K_PREP], &x.slot)) return false;
      x.flags = JG_PREPARE;
    } else {
      return false;
    }
    JRd I = J;
    I.n = pos[JG_K_ID];
    const JStr id = jr_string(I);
    gid = json_id_gid(W, J, pos[JG_K_ID], id);
  } else { /* a byteified ACCEPT: AcceptPacket :95-138 */
    gpx_wire_ref ref;
    ref.off = at;
    ref.len = len;
    WireRd r;
    WireHdr h;
    if (wr_packet(A.bytes, A.n_bytes, ref, GPX_PT_BIT(GPX_PT_ACCEPT), r, h) != GPX_WS_OK) return false;
    WireReq q;
    WireBatch B = {};
    wr_request_batch(r, q, nullptr, B);
    x.slot = wr_i32(r);
    x.bnum = wr_i32(r);
    x.bcoord = wr_i32(r);
    wr_u8(r); /* recovery */
    wr_i32(r); /* median checkpoint */
    wr_u8(r); /* noCoalesce */
    wr_i32(r); /* sender */
    if (!r.ok || r.n != r.len) return false;
    x.flags = 0;
    version = h.version;
    gid = wire_name_find(W, r.p + h.id_at, h.id_len);
  }
  GroupCtx g;
  if (wire_group(S, W, gid, version, g) != GPX_WS_OK) gid = GPX_NAME_NONE;
  return true;
}

__global__ void k_jgc_offsets(const __grid_constant__ JournalGcArgs A) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > A.n_files) return;
  const uint32_t o = A.file_off[f];
  if ((f == 0 && o != 0) || (f > 0 && o < A.file_off[f - 1]) || (f == A.n_files && o != A.n_bytes)) *A.bad_off = 1;
}

__global__ void k_jgc_parse(const __grid_constant__ DevState S, const __grid_constant__ WireNames W,
                            const __grid_constant__ JournalGcArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const uint32_t s = A.starts[i];
  JgcRec x;
  memset(&x, 0, sizeof x);
  uint32_t gid = GPX_NAME_NONE;
  bool ok = (uint64_t)s + 4u <= A.n_bytes;
  if (ok) {
    const uint32_t l = jg_be32(A.bytes + s);
    const uint64_t end = (uint64_t)s + 4u + l;
    const uint32_t f = jg_file(A, s);
    const uint32_t fend = A.file_off[f + 1];
    ok = l < 0x80000000u && end <= fend && end <= A.n_bytes;     /* inside its file */
    if (i + 1 < A.n && A.starts[i + 1] < fend) ok = ok && A.starts[i + 1] == end; /* the next frame of the file */
    if (i == 0 || A.starts[i - 1] < A.file_off[f]) ok = ok && s == A.file_off[f]; /* the file's first frame */
    if (ok) {
      x.len = l;
      ok = jg_packet(S, W, A, s + 4u, l, x, gid);
    }
  }
  if (!ok) memset(&x, 0, sizeof x);
  if (ok && gid != GPX_NAME_NONE) {
    x.gid = gid;
    x.flags |= JG_RESOLVED;
    if (jsub(x.slot, A.gc_slot[gid]) > 0) x.flags |= JG_INDEXED;
  }
  A.rec[i] = x;
  A.key[i] = (x.flags & JG_INDEXED) ? gid : S.G;
  A.cnt[(size_t)JG_UNRES * A.n + i] = ok && gid == GPX_NAME_NONE ? 1u : 0u;
  A.cnt[(size_t)JG_BAD * A.n + i] = ok ? 0u : 1u;
}

/* the keep rule: an unresolved frame is kept, a resolved one at or below its group's gc slot dropped, and a PREPARE
 * dropped when an indexed frame of its group has a higher ballot -- LogIndex.isLogMsgNeeded :336-342's test, entry by
 * entry, wrap-aware */
__global__ void k_jgc_keep(const __grid_constant__ JournalGcArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n) return;
  const JgcRec x = A.rec[i];
  bool keep = A.cnt[(size_t)JG_UNRES * A.n + i] != 0;
  if (x.flags & JG_INDEXED) {
    keep = true;
    if (x.flags & JG_PREPARE) {
      uint32_t lo = 0, hi = A.n; /* the first of the group's run */
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (A.skey[mid] < x.gid) lo = mid + 1;
        else hi = mid;
      }
      for (uint32_t j = lo; j < A.n && A.skey[j] == x.gid; j++) {
        const JgcRec e = A.rec[A.perm[j]];
        if (jsub(e.bnum, x.bnum) > 0 || (e.bnum == x.bnum && jsub(e.bcoord, x.bcoord) > 0)) {
          keep = false;
          break;
        }
      }
    }
  }
  A.cnt[(size_t)JG_KBYTES * A.n + i] = keep ? 4u + x.len : 0u;
  A.cnt[(size_t)JG_KEPT * A.n + i] = keep ? 1u : 0u;
}

__device__ __forceinline__ uint32_t jg_scanned(const JournalGcArgs& A, uint32_t row, uint32_t i) {
  return i < A.n ? A.off[(size_t)row * A.n + i] : A.tot[row];
}

/* one thread per file: a file with a torn tail, and the read-only last one, are left as they are (their frames all
 * stay); a file that keeps no frame is empty, one that drops none unchanged, any other compacted */
__global__ void k_jgc_file(const __grid_constant__ JournalGcArgs A) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= A.n_files) return;
  const uint32_t a = A.file_off[f], b = A.file_off[f + 1];
  const uint32_t lo = jg_first(A, a), hi = b > a ? jg_first(A, b) : lo;
  const uint32_t frames = hi - lo;
  const uint32_t kept = jg_scanned(A, JG_KEPT, hi) - jg_scanned(A, JG_KEPT, lo);
  const uint32_t kb_lo = jg_scanned(A, JG_KBYTES, lo);
  const uint64_t last_end = hi > lo ? (uint64_t)A.starts[hi - 1] + 4u + A.rec[hi - 1].len : a;
  JgcFile x;
  memset(&x, 0, sizeof x);
  x.lo = lo;
  x.kb_lo = kb_lo;
  x.f.unresolved = jg_scanned(A, JG_UNRES, hi) - jg_scanned(A, JG_UNRES, lo);
  x.f.kept = kept;
  x.f.dropped = frames - kept;
  if (last_end != b) x.f.status = GPX_JGC_TORN;
  else if (A.last_readonly && f + 1 == A.n_files) x.f.status = GPX_JGC_UNCHANGED;
  else if (kept == 0) x.f.status = GPX_JGC_EMPTY;
  else if (kept == frames) x.f.status = GPX_JGC_UNCHANGED;
  else x.f.status = GPX_JGC_COMPACTED;
  if (x.f.status == GPX_JGC_TORN || x.f.status == GPX_JGC_UNCHANGED) {
    x.f.kept = frames;
    x.f.dropped = 0;
  }
  if (x.f.status == GPX_JGC_COMPACTED) x.f.out_bytes = jg_scanned(A, JG_KBYTES, hi) - kb_lo;
  A.fs[f] = x;
  A.fbytes[f] = x.f.out_bytes;
}

__global__ void k_jgc_bad(const __grid_constant__ JournalGcArgs A) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < A.n && A.cnt[(size_t)JG_BAD * A.n + i]) A.bad[A.off[(size_t)JG_BAD * A.n + i]] = i;
}

__global__ void k_jgc_files(const __grid_constant__ JournalGcArgs A) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= A.n_files) return;
  gpx_journal_file x = A.fs[f].f;
  x.out_off = A.foff[f];
  A.files[f] = x;
}

#define GPX_JGC_COPY_WARPS (1u << 22) /* frames per grid-stride step of the copy */
/* thread t is lane t % 32 of the warp that copies frames t / 32, t / 32 + GPX_JGC_COPY_WARPS, ...: the bytes up to a
 * 4-byte boundary of the destination, then whole words (each lane one per 128 bytes), then the tail */
__global__ void k_jgc_copy(const __grid_constant__ JournalGcArgs A) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = (uint32_t)(t & 31u);
  for (uint64_t i = t >> 5; i < A.n; i += GPX_JGC_COPY_WARPS) {
    if (!A.cnt[(size_t)JG_KEPT * A.n + i]) continue;
    const uint32_t s = A.starts[i];
    const uint32_t f = jg_file(A, s);
    if (A.fs[f].f.status != GPX_JGC_COMPACTED) continue;
    const uint8_t* src = A.bytes + s;
    uint8_t* dst = A.out + A.foff[f] + (A.off[(size_t)JG_KBYTES * A.n + i] - A.fs[f].kb_lo);
    const uint32_t L = 4u + A.rec[i].len;
    const uint32_t head = min(L, (uint32_t)((4u - ((size_t)dst & 3u)) & 3u));
    for (uint32_t b = lane; b < head; b += 32) dst[b] = src[b];
    const uint32_t nw = (L - head) >> 2;
    uint32_t* dw = reinterpret_cast<uint32_t*>(dst + head);
    const uint8_t* sw = src + head;
    for (uint32_t w = lane; w < nw; w += 32) {
      const uint8_t* q = sw + 4u * w;
      dw[w] = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
    }
    for (uint32_t b = head + 4u * nw + lane; b < L; b += 32) dst[b] = src[b];
  }
}
