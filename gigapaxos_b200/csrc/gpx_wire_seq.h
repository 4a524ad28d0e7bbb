/* gpx_wire_seq.h -- the host sequence of every wire and response-cache call: the argument checks, the scratch layouts,
 * the passes, sorts, scans and gathers between the scalar kernels, the capacity decision and the early exits.  Each
 * sequence is written once, as a function template over an executor, and holds no CUDA syntax, so nvcc compiles it
 * into the product (gpx_wire_host.inc, gpx_respcache_host.inc: the CUDA executor) and g++ into the CPU tests
 * (tests/emu: the CPU executor).  Included by gpx_engine.cu once fail() is defined; the tests define their own.
 *
 * An executor `ex` does only what differs between the device and the host:
 *   ex.launch(kernel, n, block, args...)      kernel(args...) over n threads in blocks of `block`
 *   ex.sort(key, skey, val, perm, n, bits, tmp, tmp_bytes)
 *                                             stable pair sort of n 32- or 64-bit keys on their low `bits` bits
 *   ex.scan(cnt, off, n, rows, scan[, bound]) exclusive prefix sums of `rows` rows of n counters each; the CPU executor
 *                                             also checks each row's total against bound
 *   ex.totals(cnt, off, n, rows, tot)         the rows' totals into tot (scratch)
 *   ex.scan_by_key(key, sum, pre, n, scan)    JsonCompose's exclusive scan by key
 *   ex.sum_by_key(key, val, start, n, scan)   exclusive sum by 64-bit key
 *   ex.fill(p, byte, bytes), ex.upload(dst, host, bytes), ex.column(dst, src, pitch, n)
 *                                             memset; copy from host memory; dst[i] = the word at src + i * pitch
 *   ex.read(host, src, bytes), ex.sync()      copy to host memory, there once sync() returns
 *   ex.grow(&buf, &cap, bytes, keep)          buf holds at least `bytes`, its first `keep` bytes kept
 *   ex.scan_bytes(n), ex.sort_bytes(n, bits), ex.sort64_bytes(n, bits), ex.scan_by_key_bytes(n),
 *   ex.sum_by_key_bytes(n)                    the temporary storage each of those needs
 * Every operation returns GPX_OK or an error code except the sizes.  A call object `call` has begin() and end(), the
 * engine's ordering between calls: begin() runs once the arguments pass, before any device work, and may create the
 * name table and the recipient sets that WireEnv::W and the sweep's Z refer to. */
#pragma once

#include <algorithm>
#include <cstring>

#include "gpx_journal.cuh"
#include "gpx_journal_gc.cuh"
#include "gpx_respcache.cuh"
#include "gpx_wire_dev.cuh"
#include "gpx_wire_fwd.cuh"
#include "gpx_wire_json.cuh"
#include "gpx_wire_json_enc.cuh"

/* what a sequence works on: the engine's state and name table, read by reference, and its scratch buffer */
struct WireEnv {
  const DevState& S;
  const WireNames& W;
  void** buf;
  size_t* bytes;
};

/* carves 256-byte aligned pieces out of one allocation; over base == nullptr it only sums the sizes */
struct Carve {
  uint8_t* base;
  size_t used = 0;
  template <typename T>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
    used += (n * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};

/* lays a scratch layout out over *buf: over nullptr to size it, then over *buf grown to that size.  The layout returns
 * how many of its leading bytes an earlier pass has filled; a reallocation moves them along. */
template <class Ex, typename Layout>
static int wire_place(Ex& ex, void** buf, size_t* cap, Layout&& layout) {
  Carve c{nullptr};
  const size_t keep = layout(c);
  int rc = ex.grow(buf, cap, c.used, keep);
  if (rc) return rc;
  c = Carve{(uint8_t*)*buf};
  layout(c);
  return GPX_OK;
}

static int key_bits(uint64_t max_key) {
  int b = 1;
  while (b < 32 && (1ull << b) <= max_key) b++;
  return b;
}
template <class Ex>
static size_t wire_cub_bytes(Ex& ex, uint32_t n, int key_bits) {
  return std::max(ex.scan_bytes(n), ex.sort_bytes(n, key_bits));
}

/* one output of a wire call: its size is the caller's capacity going in and the size the call needs coming out */
struct WireOut {
  uint32_t* n32 = nullptr;
  uint64_t* n64 = nullptr;
  bool given; /* the output buffer is there */
  uint64_t cap = 0;
  WireOut(uint32_t* n, bool given) : n32(n), given(given) {}
  WireOut(uint64_t* n, bool given) : n64(n), given(given) {}
  void set(uint64_t v) const {
    if (n32) *n32 = (uint32_t)v;
    else *n64 = v;
  }
};

/* what every wire call checks first, in this order: null arguments (GPX_EINVAL; `inputs` is false when an input is
 * missing), then n_bytes (GPX_ERANGE).  Then it reads the capacities and zeroes the sizes. */
template <size_t K>
static int wire_args(bool inputs, uint64_t n_bytes, WireOut (&o)[K]) {
  bool sizes = true;
  for (const WireOut& x : o) sizes = sizes && (x.n32 || x.n64);
  if (!sizes || !inputs) return fail(GPX_EINVAL, "null argument");
  if (n_bytes > 0xffffffffull) return fail(GPX_ERANGE, "n_bytes > 4 GiB");
  for (WireOut& x : o) {
    x.cap = x.n32 ? *x.n32 : *x.n64;
    x.set(0);
  }
  return GPX_OK;
}

/* the sizes tot[K] out; GPX_ERANGE when an output is too small (nothing is written then), else GPX_EINVAL when an
 * output that is needed is null */
template <size_t K>
static int wire_fit(const WireOut (&o)[K], const uint32_t* tot, const char* too_small) {
  bool small = false, null = false;
  for (size_t j = 0; j < K; j++) {
    o[j].set(tot[j]);
    small = small || tot[j] > o[j].cap;
    null = null || (tot[j] && !o[j].given);
  }
  if (small) return fail(GPX_ERANGE, too_small);
  return null ? fail(GPX_EINVAL, "null output") : GPX_OK;
}

template <typename T>
struct Gather {
  const T* src;
  T* dst;
};
template <typename T>
static Gather<T> gather(const T* src, T* dst) {
  return {src, dst};
}

/* a stable sort by gid of up to `cap` items, [iota | perm | skeys | cub], and the gathers into its order */
struct GidSort {
  uint32_t cap;
  int kb; /* the key bits of max_groups */
  size_t cub_bytes;
  uint32_t *iota = nullptr, *perm = nullptr, *skeys = nullptr;
  void* cub = nullptr;
  bool counted = false; /* iota holds 0 .. cap-1 */
  template <class Ex>
  GidSort(Ex& ex, uint32_t cap, uint32_t max_groups)
      : cap(cap), kb(key_bits(max_groups)), cub_bytes(wire_cub_bytes(ex, cap, kb)) {}
  void lay(Carve& c) {
    iota = c.take<uint32_t>(cap);
    perm = c.take<uint32_t>(cap);
    skeys = c.take<uint32_t>(cap);
    cub = c.take<uint8_t>(cub_bytes);
  }
  /* sorts the first n keys, then dst[i] = src[perm[i]] for every output.  Left in flight. */
  template <class Ex, typename... T>
  int run(Ex& ex, const uint32_t* key, uint32_t n, Gather<T>... outs) {
    if (n == 0) return GPX_OK;
    int rc;
    if (!counted) {
      if ((rc = ex.launch(k_wire_iota, cap, 256, iota, cap))) return rc;
      counted = true;
    }
    if ((rc = ex.sort(key, skeys, iota, perm, n, kb, cub, cub_bytes))) return rc;
    (void)((rc = ex.launch(k_wire_gather<T>, n, 256, outs.src, (const uint32_t*)perm, n, outs.dst)) || ...);
    return rc;
  }
};

/* the scans of a counting pass: the totals of its counter rows and the scans' temporary storage */
struct WireScan {
  size_t cub_bytes;
  uint32_t* tot = nullptr;
  void* cub = nullptr;
  void lay(Carve& c, uint32_t rows) {
    tot = c.take<uint32_t>(rows);
    cub = c.take<uint8_t>(cub_bytes);
  }
};

/* exclusive prefix sums of `rows` arrays of n counters each, in place into `off`; the totals reach h_tot[rows] once
 * the caller synchronises */
template <class Ex>
static int wire_scan(Ex& ex, const uint32_t* cnt, uint32_t* off, uint32_t n, uint32_t rows, const WireScan& s,
                     uint32_t* h_tot) {
  int rc;
  if ((rc = ex.scan(cnt, off, n, rows, s)) || (rc = ex.totals(cnt, off, n, rows, s.tot))) return rc;
  return ex.read(h_tot, s.tot, rows * 4ull);
}

/* a decoder's pass 0 counters [cnt | off]: `rows` counters per packet and their prefix sums, which pass 1 keeps */
static size_t wire_counters(Carve& c, uint32_t rows, uint32_t n, uint32_t** cnt, uint32_t** off) {
  *cnt = c.take<uint32_t>((size_t)rows * n);
  *off = c.take<uint32_t>((size_t)rows * n);
  return c.used;
}
/* a decoder's pass 0 scratch: the counters and their scans */
static size_t wire_count_pass(Carve& c, uint32_t rows, uint32_t n, uint32_t** cnt, uint32_t** off, WireScan& scan) {
  wire_counters(c, rows, n, cnt, off);
  scan.lay(c, rows);
  return 0;
}

/* a decoder's packets are there: their refs, statuses and (when it has bytes) the arena */
static bool wire_packets_given(uint32_t n, const uint8_t* bytes, uint64_t n_bytes, const gpx_wire_ref* pkts,
                               const int32_t* status) {
  return n == 0 || (pkts && status && (bytes || !n_bytes));
}

/* ---- decode ---------------------------------------------------------------------------------------------------- */
/* k_wire_decode's pass 1 scratch: pass 0's counters, the records staged in packet order, their sort keys (gids) and
 * the sort */
static size_t decode_pass1(Carve& c, WireDecodeArgs& A, const uint32_t* tot, GidSort& sort) {
  const size_t keep = wire_counters(c, WD_NCNT, A.n, &A.cnt, &A.off);
  A.acc = c.take<gpx_accept_rec>(tot[WD_ACC]);
  A.rep = c.take<gpx_accept_reply_rec>(tot[WD_REP]);
  A.dec = c.take<gpx_decision_rec>(tot[WD_DEC]);
  A.acc_key = c.take<uint32_t>(tot[WD_ACC]);
  A.rep_key = c.take<uint32_t>(tot[WD_REP]);
  A.dec_key = c.take<uint32_t>(tot[WD_DEC]);
  sort.lay(c);
  return keep;
}

static WireDecodeArgs decode_args(uint32_t n, const uint8_t* bytes, uint64_t n_bytes, const gpx_wire_ref* pkts,
                                  int32_t* status) {
  WireDecodeArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.n_bytes = n_bytes;
  A.n = n;
  A.status = status;
  return A;
}

/* pass 0: A.status, the packets' output sizes and their prefix sums; the totals reach h_tot once the caller
 * synchronises.  A carries bytes, pkts, n_bytes, n and status. */
template <class Ex>
static int wire_decode_count(Ex& ex, const WireEnv& E, WireDecodeArgs& A, uint32_t* h_tot) {
  WireScan scan{wire_cub_bytes(ex, A.n, key_bits(E.S.G))};
  int rc = wire_place(ex, E.buf, E.bytes,
                      [&](Carve& c) { return wire_count_pass(c, WD_NCNT, A.n, &A.cnt, &A.off, scan); });
  if (rc) return rc;
  A.emit = 0;
  if ((rc = ex.launch(k_wire_decode, A.n, 128, E.S, E.W, A))) return rc;
  return wire_scan(ex, A.cnt, A.off, A.n, WD_NCNT, scan, h_tot);
}

/* pass 1: the records in packet order into scratch behind the scanned offsets, the request bodies straight into blob;
 * then per record type a stable sort by gid and a gather straight into its output.  Left in flight. */
template <class Ex>
static int wire_decode_emit(Ex& ex, const WireEnv& E, WireDecodeArgs& A, const uint32_t* tot, gpx_accept_rec* accepts,
                            uint8_t* blob, gpx_accept_reply_rec* replies, gpx_decision_rec* decisions) {
  GidSort sort(ex, std::max(tot[WD_ACC], std::max(tot[WD_REP], tot[WD_DEC])), E.S.G);
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) { return decode_pass1(c, A, tot, sort); });
  if (rc) return rc;
  A.blob = blob;
  A.emit = 1;
  if ((rc = ex.launch(k_wire_decode, A.n, 128, E.S, E.W, A))) return rc;
  /* replies and decisions are 32-byte pvalue headers */
  if ((rc = sort.run(ex, A.acc_key, tot[WD_ACC], gather(A.acc, accepts))) ||
      (rc = sort.run(ex, A.rep_key, tot[WD_REP], gather((const gpx_pvalue_hdr*)A.rep, (gpx_pvalue_hdr*)replies))))
    return rc;
  return sort.run(ex, A.dec_key, tot[WD_DEC], gather((const gpx_pvalue_hdr*)A.dec, (gpx_pvalue_hdr*)decisions));
}

/* gpx_wire_decode_batch_device */
template <class Ex, class C>
static int wire_decode(Ex& ex, C& call, const WireEnv& E, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                       const gpx_wire_ref* pkts, int32_t* status, gpx_accept_rec* accepts, uint32_t* n_accepts,
                       uint8_t* blob, uint64_t* blob_bytes, gpx_accept_reply_rec* replies, uint32_t* n_replies,
                       gpx_decision_rec* decisions, uint32_t* n_decisions) {
  WireOut o[] = {{n_accepts, accepts != nullptr}, {blob_bytes, blob != nullptr}, {n_replies, replies != nullptr},
                 {n_decisions, decisions != nullptr}};
  int rc = wire_args(wire_packets_given(n, bytes, n_bytes, pkts, status), n_bytes, o);
  if (rc || n == 0) return rc;
  if ((rc = call.begin())) return rc;
  WireDecodeArgs A = decode_args(n, bytes, n_bytes, pkts, status);
  uint32_t tot[WD_NCNT];
  if ((rc = wire_decode_count(ex, E, A, tot))) return rc;
  if ((rc = ex.sync())) return rc; /* the one host read: the radix sorts need the item counts */
  if ((rc = wire_fit(o, tot, "decode output too small"))) return rc;
  if ((rc = wire_decode_emit(ex, E, A, tot, accepts, blob, replies, decisions))) return rc;
  return call.end();
}

/* ---- encode ---------------------------------------------------------------------------------------------------- */
enum WireEnc { ENC_REPLIES, ENC_DECISIONS, ENC_ACCEPTS };

/* the keys kernel (keys) or a pass of the encoder `kind` over A.n records; Q carries the ACCEPTs' requests */
template <class Ex>
static int wire_enc_launch(Ex& ex, const WireEnv& E, WireEnc kind, bool keys, const WireEncodeArgs& A,
                           const WireAccArgs& Q) {
  const uint32_t b = keys ? 256 : 128;
  switch (kind) {
    case ENC_REPLIES:
      return keys ? ex.launch(k_wire_enc_keys_replies, A.n, b, E.S, E.W, A)
                  : ex.launch(k_wire_enc_replies, A.n, b, E.S, E.W, A);
    case ENC_DECISIONS:
      return keys ? ex.launch(k_wire_enc_keys_decisions, A.n, b, E.S, E.W, A)
                  : ex.launch(k_wire_enc_decisions, A.n, b, E.S, E.W, A);
    case ENC_ACCEPTS:
      return keys ? ex.launch(k_wire_enc_keys_accepts, A.n, b, E.S, E.W, A, Q)
                  : ex.launch(k_wire_enc_accepts, A.n, b, E.S, E.W, A, Q);
  }
  return GPX_OK;
}

/* the encoders' scratch: the keys and their stable sort [key | iota | perm | skey], which the passes read, then pass
 * 0's counters [cnt | off] and their scans */
struct EncodeScratch {
  uint32_t n;
  WireScan scan;
  uint32_t *key, *iota, *perm, *skey, *cnt, *off;
  size_t lay(Carve& c) {
    key = c.take<uint32_t>(n);
    iota = c.take<uint32_t>(n);
    perm = c.take<uint32_t>(n);
    skey = c.take<uint32_t>(n);
    cnt = c.take<uint32_t>(2ull * n);
    off = c.take<uint32_t>(2ull * n);
    scan.lay(c, 2);
    return 0;
  }
};

/* the keys, the stable sort, pass 0 and the scans: rstatus into A.rstatus, the totals (packet bytes, index entries)
 * reach h_tot once the caller synchronises.  A carries recs, n, n_lanes, rstatus and n_ptr; the sort and the offsets
 * live in the scratch for pass 1. */
template <class Ex>
static int wire_encode_count(Ex& ex, const WireEnv& E, WireEnc kind, WireEncodeArgs& A, const WireAccArgs& Q,
                             uint32_t* h_tot) {
  const uint32_t n = A.n;
  EncodeScratch s{n, {wire_cub_bytes(ex, n, 32)}}; /* GPX_WIRE_NOKEY is all ones: all 32 key bits are sorted */
  int rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) { return s.lay(c); });
  if (rc) return rc;
  A.key = s.key;
  A.perm = s.perm;
  A.skey = s.skey;
  A.cnt = s.cnt;
  A.off = s.off;
  if ((rc = wire_enc_launch(ex, E, kind, true, A, Q)) || (rc = ex.launch(k_wire_iota, n, 256, s.iota, n)) ||
      /* the records that are not encoded (GPX_WIRE_NOKEY) sort last */
      (rc = ex.sort((const uint32_t*)A.key, s.skey, s.iota, s.perm, n, 32, s.scan.cub, s.scan.cub_bytes)))
    return rc;
  A.emit = 0;
  if ((rc = wire_enc_launch(ex, E, kind, false, A, Q))) return rc;
  return wire_scan(ex, s.cnt, s.off, n, 2, s.scan, h_tot);
}

static WireEncodeArgs encode_args(uint32_t n_lanes, uint32_t n, const uint32_t* n_ptr, const void* recs,
                                  uint8_t* rstatus) {
  WireEncodeArgs A;
  memset(&A, 0, sizeof A);
  A.recs = recs;
  A.n = n;
  A.n_lanes = n_lanes;
  A.rstatus = rstatus;
  A.n_ptr = n_ptr;
  return A;
}

/* the checks every encoder makes before it runs: null arguments, the output capacities in; n % n_lanes for replies */
static int wire_encode_args(WireEnc kind, uint32_t n_lanes, uint32_t n, const void* recs, const uint8_t* rstatus,
                            WireOut (&o)[2]) {
  int rc = wire_args(!n || (recs && rstatus), 0, o);
  if (rc || n == 0) return rc;
  if (kind == ENC_REPLIES && n % n_lanes) return fail(GPX_EINVAL, "replies: n is not a multiple of n_lanes");
  return GPX_OK;
}

/* the device-buffer encoders; n_ptr (decisions, accepts) is a device count of the records, at most n */
template <class Ex, class C>
static int wire_encode(Ex& ex, C& call, const WireEnv& E, WireEnc kind, uint32_t n, const uint32_t* n_ptr,
                       const void* recs, const WireAccArgs& Q, uint8_t* rstatus, uint8_t* out, uint64_t* out_bytes,
                       gpx_wire_ref* refs, uint32_t* n_refs) {
  if (kind == ENC_ACCEPTS && n && (!Q.head || (Q.n_reqs && (!Q.reqs || !Q.meta || !Q.payload))))
    return fail(GPX_EINVAL, "null argument");
  WireOut o[] = {{out_bytes, out != nullptr}, {n_refs, refs != nullptr}};
  int rc = wire_encode_args(kind, E.S.L, n, recs, rstatus, o);
  if (rc || n == 0) return rc;
  if ((rc = call.begin())) return rc;
  WireEncodeArgs A = encode_args(E.S.L, n, n_ptr, recs, rstatus);
  uint32_t tot[2];
  if ((rc = wire_encode_count(ex, E, kind, A, Q, tot))) return rc;
  if ((rc = ex.sync())) return rc; /* the one host read: the output sizes */
  if ((rc = wire_fit(o, tot, "encode output too small"))) return rc;
  if (tot[0] == 0) return GPX_OK;
  /* pass 1: the packets and their index entries at the scanned offsets, left in flight */
  A.out = out;
  A.refs = refs;
  A.emit = 1;
  if ((rc = wire_enc_launch(ex, E, kind, false, A, Q))) return rc;
  return call.end();
}

/* ---- REQUEST packets -> proposals ---------------------------------------------------------------------------------- */
/* the requests decoders' pass 1 scratch: pass 0's counters, the requests and meta staged in packet (member) order,
 * their sort keys (gids) and the sort.  Args: WireReqDecodeArgs or WireJsonReqArgs. */
template <typename Args>
static size_t requests_pass1(Carve& c, Args& A, uint32_t nq, GidSort& sort) {
  uint32_t* off;
  const size_t keep = wire_counters(c, WQ_NCNT, A.n, &A.cnt, &off);
  A.off = off;
  A.req = c.take<gpx_request_rec>(nq);
  A.meta = c.take<gpx_wire_req_meta>(nq);
  A.key = c.take<uint32_t>(nq);
  sort.lay(c);
  return keep;
}

/* the two passes of a requests decoder's kernel k over A.n items (packets or members).  A carries the inputs, now_ms
 * and status; the outputs are grouped by gid. */
template <class Ex, class C, typename Args>
static int wire_requests_run(Ex& ex, C& call, const WireEnv& E, void (*k)(DevState, WireNames, Args), Args& A,
                             WireOut (&o)[2], gpx_request_rec* reqs, gpx_wire_req_meta* meta, uint8_t* payload) {
  const uint32_t n = A.n;
  int rc;
  if ((rc = call.begin())) return rc;
  WireScan scan{wire_cub_bytes(ex, n, key_bits(E.S.G))};
  uint32_t* off;
  if ((rc = wire_place(ex, E.buf, E.bytes,
                       [&](Carve& c) { return wire_count_pass(c, WQ_NCNT, n, &A.cnt, &off, scan); })))
    return rc;
  A.off = off;
  A.emit = 0;
  if ((rc = ex.launch(k, n, 128, E.S, E.W, A))) return rc;
  uint32_t tot[WQ_NCNT];
  if ((rc = wire_scan(ex, A.cnt, off, n, WQ_NCNT, scan, tot))) return rc;
  if ((rc = ex.sync())) return rc; /* the one host read: the radix sort needs the item count */
  if ((rc = wire_fit(o, tot, "decode output too small"))) return rc;
  const uint32_t nq = tot[WQ_REQ];
  if (nq == 0) return call.end();
  /* pass 1: requests and meta staged in input order behind the offsets, then a stable sort by gid and the gathers */
  GidSort sort(ex, nq, E.S.G);
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) { return requests_pass1(c, A, nq, sort); }))) return rc;
  A.payload = payload;
  A.emit = 1;
  if ((rc = ex.launch(k, n, 128, E.S, E.W, A))) return rc;
  if ((rc = sort.run(ex, A.key, nq, gather(A.req, reqs), gather(A.meta, meta)))) return rc;
  return call.end();
}

/* gpx_wire_decode_requests_device */
template <class Ex, class C>
static int wire_decode_requests(Ex& ex, C& call, const WireEnv& E, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                const gpx_wire_ref* pkts, int64_t now_ms, int32_t* status, gpx_request_rec* reqs,
                                gpx_wire_req_meta* meta, uint32_t* n_reqs, uint8_t* payload, uint64_t* payload_bytes) {
  WireOut o[] = {{n_reqs, reqs && meta}, {payload_bytes, payload != nullptr}};
  int rc = wire_args(wire_packets_given(n, bytes, n_bytes, pkts, status), n_bytes, o);
  if (rc || n == 0) return rc;
  WireReqDecodeArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.n_bytes = n_bytes;
  A.n = n;
  A.now_ms = now_ms;
  A.status = status;
  return wire_requests_run(ex, call, E, k_wire_req_decode, A, o, reqs, meta, payload);
}

/* gpx_wire_decode_json_requests_device */
template <class Ex, class C>
static int wire_decode_json_requests(Ex& ex, C& call, const WireEnv& E, uint32_t n_members, const uint8_t* bytes,
                                     uint64_t n_bytes, const gpx_wire_ref* pkts, uint32_t n_pkts,
                                     const gpx_wire_member* members, int64_t now_ms, int32_t* status,
                                     gpx_request_rec* reqs, gpx_wire_req_meta* meta, uint32_t* n_reqs,
                                     uint8_t* payload, uint64_t* payload_bytes) {
  WireOut o[] = {{n_reqs, reqs && meta}, {payload_bytes, payload != nullptr}};
  const bool given = !n_members || (members && status && (bytes || !n_bytes) && (pkts || !n_pkts));
  int rc = wire_args(given, n_bytes, o);
  if (rc || n_members == 0) return rc;
  WireJsonReqArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.mem = members;
  A.n_bytes = n_bytes;
  A.n_pkts = n_pkts;
  A.n = n_members;
  A.now_ms = now_ms;
  A.status = status;
  return wire_requests_run(ex, call, E, k_json_req, A, o, reqs, meta, payload);
}

/* gpx_wire_decode_client_requests_device: the packets are the members */
template <class Ex, class C>
static int wire_decode_client_requests(Ex& ex, C& call, const WireEnv& E, uint32_t n, const uint8_t* bytes,
                                       uint64_t n_bytes, const gpx_wire_ref* pkts, const gpx_wire_peer* peers,
                                       int64_t now_ms, int32_t* status, gpx_request_rec* reqs, gpx_wire_req_meta* meta,
                                       uint32_t* n_reqs, uint8_t* payload, uint64_t* payload_bytes) {
  WireOut o[] = {{n_reqs, reqs && meta}, {payload_bytes, payload != nullptr}};
  int rc = wire_args(wire_packets_given(n, bytes, n_bytes, pkts, status), n_bytes, o);
  if (rc || n == 0) return rc;
  WireClientReqArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.peers = peers;
  A.n_bytes = n_bytes;
  A.n_pkts = n;
  A.n = n;
  A.now_ms = now_ms;
  A.status = status;
  return wire_requests_run(ex, call, E, k_json_client, A, o, reqs, meta, payload);
}

/* ---- forwards: a non-coordinator's REQUEST packets (gpx_wire_fwd.cuh) ------------------------------------------------ */
template <class Ex, class C>
static int wire_encode_forwards(Ex& ex, C& call, const WireEnv& E, const gpx_request_rec* reqs,
                                const gpx_wire_req_meta* meta, uint32_t n, const int32_t* status,
                                const uint8_t* payload, uint32_t n_down, const int32_t* down_nodes, uint8_t* rstatus,
                                uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs, uint32_t* n_refs) {
  WireOut o[] = {{out_bytes, out != nullptr}, {n_refs, refs != nullptr}};
  int rc = wire_args((!n || (reqs && meta && status && payload && rstatus)) && (!n_down || down_nodes), 0, o);
  if (rc || n == 0) return rc;
  if ((rc = call.begin())) return rc;
  WireFwdArgs A;
  memset(&A, 0, sizeof A);
  A.reqs = reqs;
  A.meta = meta;
  A.status = status;
  A.payload = payload;
  A.n = n;
  A.n_down = n_down;
  A.rstatus = rstatus;
  /* pass 0's counters and scans, and the down nodes */
  WireScan scan{wire_cub_bytes(ex, n, key_bits(E.S.G))};
  uint32_t* off;
  int32_t* down;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
         wire_count_pass(c, 2, n, &A.cnt, &off, scan);
         down = c.take<int32_t>(n_down);
         return (size_t)0;
       })))
    return rc;
  if (n_down && (rc = ex.upload(down, down_nodes, n_down * 4ull))) return rc;
  A.down = down;
  A.off = off;
  A.emit = 0;
  if ((rc = ex.launch(k_wire_fwd, n, 128, E.S, E.W, A))) return rc;
  uint32_t tot[2];
  if ((rc = wire_scan(ex, A.cnt, off, n, 2, scan, tot))) return rc;
  if ((rc = ex.sync())) return rc; /* the one host read: the output sizes */
  if ((rc = wire_fit(o, tot, "encode output too small"))) return rc;
  if (tot[1] == 0) return GPX_OK;
  /* pass 1: the packets and their refs at the scanned offsets, left in flight */
  A.out = out;
  A.refs = refs;
  A.emit = 1;
  if ((rc = ex.launch(k_wire_fwd, n, 128, E.S, E.W, A))) return rc;
  return call.end();
}

/* ---- JSON replies and commits (gpx_wire_json.cuh) --------------------------------------------------------------------
 * Every size before the one synchronisation is a bound the host knows: chunks n_bytes / GPX_JSON_CHUNK + 2n (when the
 * packets' lengths add up to at most n_bytes), events (depth-3 opens, depth-1 closes) half the bytes those chunks cover
 * + n each, members a GPX_JSON_MIN_MEMBER-th + n.  The kernels that run over a count only the device knows read it
 * there and leave the slots past it inert. */
template <class Ex>
static size_t json_cub_bytes(Ex& ex, uint32_t n) {
  return std::max(ex.scan_bytes(n), ex.scan_by_key_bytes(n));
}

/* the JSON decoder's scratch.  The packets' and members' arrays [pcnt | poff | bad | pp | mcnt | moff | mem] lead and
 * live on into pass 1; pass 0 adds the chunks, the events and the scans, pass 1 the records staged in member order,
 * their sort keys (gids) and the sort. */
static size_t json_kept(Carve& c, WireJsonArgs& A) {
  A.pcnt = c.take<uint32_t>(2ull * A.n);
  A.poff = c.take<uint32_t>(2ull * A.n);
  A.bad = c.take<uint32_t>(A.n);
  A.pp = c.take<uint32_t>(3ull * A.n);
  A.mcnt = c.take<uint32_t>(3ull * A.cap_mem);
  A.moff = c.take<uint32_t>(3ull * A.cap_mem);
  A.mem = c.take<gpx_wire_member>(A.cap_mem);
  return c.used;
}
static size_t json_pass0(Carve& c, WireJsonArgs& A, uint32_t cap_ev, WireScan& scan) {
  json_kept(c, A);
  A.ikey = c.take<uint32_t>(A.cap_items);
  A.isum = c.take<JsonSum>(A.cap_items);
  A.ipre = c.take<JsonSum>(A.cap_items);
  A.ecnt = c.take<uint32_t>(2ull * A.cap_items);
  A.eoff = c.take<uint32_t>(2ull * A.cap_items);
  A.ev_open = c.take<uint32_t>(cap_ev);
  A.ev_close = c.take<uint32_t>(cap_ev);
  scan.lay(c, 8);
  return 0;
}
static size_t json_pass1(Carve& c, WireJsonArgs& A, uint32_t nr, uint32_t nd, GidSort& sort) {
  const size_t keep = json_kept(c, A);
  A.rep = c.take<gpx_accept_reply_rec>(nr);
  A.dec = c.take<gpx_decision_rec>(nd);
  A.rep_key = c.take<uint32_t>(nr);
  A.dec_key = c.take<uint32_t>(nd);
  sort.lay(c);
  return keep;
}

/* gpx_wire_decode_json_device */
template <class Ex, class C>
static int wire_decode_json(Ex& ex, C& call, const WireEnv& E, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                            const gpx_wire_ref* pkts, int32_t* status, gpx_wire_member* members, uint32_t* n_members,
                            gpx_accept_reply_rec* replies, uint32_t* n_replies, gpx_decision_rec* decisions,
                            uint32_t* n_decisions) {
  WireOut o[] = {{n_members, members != nullptr}, {n_replies, replies != nullptr}, {n_decisions, decisions != nullptr}};
  int rc = wire_args(wire_packets_given(n, bytes, n_bytes, pkts, status), n_bytes, o);
  if (rc || n == 0) return rc;
  if ((rc = call.begin())) return rc;
  const uint64_t cap_items64 = n_bytes / GPX_JSON_CHUNK + 2ull * n + 1ull;
  const uint64_t cap_ev64 = cap_items64 * GPX_JSON_CHUNK / 2ull + n + 1ull;
  const uint64_t cap_mem64 = cap_items64 * GPX_JSON_CHUNK / GPX_JSON_MIN_MEMBER + n + 1ull;
  if (cap_ev64 > 0x7fffffffull || cap_mem64 > 0x7fffffffull) return fail(GPX_ERANGE, "batch too large");
  const uint32_t cap_items = (uint32_t)cap_items64, cap_ev = (uint32_t)cap_ev64, cap_mem = (uint32_t)cap_mem64;
  WireScan scan{std::max(json_cub_bytes(ex, std::max(cap_items, cap_mem)), json_cub_bytes(ex, n))};
  WireJsonArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.n_bytes = n_bytes;
  A.n = n;
  A.status = status;
  A.cap_items = cap_items;
  A.cap_mem = cap_mem;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) { return json_pass0(c, A, cap_ev, scan); }))) return rc;
  /* pass 0: structure, packets, members; the sizes.  The bounds on the events and the members are the arrays' sizes
   * the kernels write into; the device keeps them, the CPU executor's scans check them. */
  if ((rc = ex.launch(k_json_pre, n, 128, A)) || (rc = ex.scan(A.pcnt, A.poff, n, 1, scan)) ||
      (rc = ex.launch(k_json_sum, cap_items, 128, A)) ||
      (rc = ex.scan_by_key(A.ikey, A.isum, A.ipre, cap_items, scan)))
    return rc;
  A.emit = 0;
  if ((rc = ex.launch(k_json_struct, cap_items, 128, A)) || (rc = ex.scan(A.ecnt, A.eoff, cap_items, 2, scan, cap_ev)))
    return rc;
  A.emit = 1;
  if ((rc = ex.launch(k_json_struct, cap_items, 128, A)) || (rc = ex.launch(k_json_packet, n, 128, A)) ||
      (rc = ex.scan(A.pcnt + n, A.poff + n, n, 1, scan, cap_mem)))
    return rc;
  A.emit = 0;
  if ((rc = ex.launch(k_json_member, cap_mem, 128, E.S, E.W, A)) ||
      (rc = ex.launch(k_json_fix, std::max(n, cap_mem), 256, A)) ||
      (rc = ex.scan(A.mcnt, A.moff, cap_mem, 3, scan)) || (rc = ex.totals(A.pcnt, A.poff, n, 2, scan.tot)) ||
      (rc = ex.totals(A.mcnt, A.moff, cap_mem, 3, scan.tot + 2)))
    return rc;
  uint32_t tot[5];
  if ((rc = ex.read(tot, scan.tot, sizeof tot)) || (rc = ex.sync())) return rc; /* the one host read: the sizes */
  if (tot[0] > cap_items || tot[1] > cap_mem) return fail(GPX_EINVAL, "packet lengths add up to more than n_bytes");
  if ((rc = wire_fit(o, tot + 2, "decode output too small"))) return rc;
  const uint32_t nm = tot[2], nr = tot[3], nd = tot[4];
  if (nm == 0) return call.end();
  /* pass 1: members and records in member order, then per record type a stable sort by gid and the gather */
  GidSort sort(ex, std::max(nr, nd), E.S.G);
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) { return json_pass1(c, A, nr, nd, sort); }))) return rc;
  /* the event lists are gone with the rest of pass 0's scratch: pass 1 finds wrapper members by their off */
  A.ev_open = nullptr;
  A.mem_out = members;
  A.emit = 1;
  if ((rc = ex.launch(k_json_member, tot[1], 128, E.S, E.W, A)) ||
      (rc = sort.run(ex, A.rep_key, nr, gather((const gpx_pvalue_hdr*)A.rep, (gpx_pvalue_hdr*)replies))) ||
      (rc = sort.run(ex, A.dec_key, nd, gather((const gpx_pvalue_hdr*)A.dec, (gpx_pvalue_hdr*)decisions))))
    return rc;
  return call.end();
}

/* ---- the JSON form on the sending side (gpx_wire_json_enc.cuh) ------------------------------------------------------- */
template <class Ex>
static size_t json_enc_cub_bytes(Ex& ex, uint32_t nr, uint32_t nd, uint32_t n) {
  const size_t a = std::max(wire_cub_bytes(ex, std::max(nr, nd), 32), wire_cub_bytes(ex, n, 32));
  return std::max(a, std::max(ex.sort64_bytes(n, 35), ex.sum_by_key_bytes(n)));
}

/* gpx_wire_encode_json_sweep_device; gpx_wire_encode_json_device is the sweep without forwards.  Z: the recipient
 * sets, which call.begin() brings up to date */
template <class Ex, class C>
static int wire_encode_json_sweep(Ex& ex, C& call, const WireEnv& E, const JsonSets& Z, uint32_t n_replies,
                                  const gpx_accept_reply_rec* replies, const gpx_decision_rec* decisions,
                                  const uint32_t* n_dec_ptr, uint32_t n_dec_max, const gpx_request_rec* reqs,
                                  const gpx_wire_req_meta* meta, uint32_t n_reqs, const int32_t* status,
                                  const uint8_t* payload, uint32_t n_down, const int32_t* down_nodes,
                                  uint8_t* rstatus_replies, uint8_t* rstatus_decisions, uint8_t* rstatus_reqs,
                                  uint64_t wrap_bytes, uint8_t* out, uint64_t* out_bytes, gpx_wire_ref* refs,
                                  uint32_t* n_refs) {
  WireOut o[] = {{out_bytes, out != nullptr}, {n_refs, refs != nullptr}};
  const bool given = (!n_replies || (replies && rstatus_replies)) && (!n_dec_max || (decisions && rstatus_decisions)) &&
                     (!n_reqs || (reqs && meta && status && payload && rstatus_reqs)) && (!n_down || down_nodes);
  int rc = wire_args(given, 0, o);
  if (rc) return rc;
  if (wrap_bytes == 0) wrap_bytes = GPX_JSON_WRAP_BYTES;
  if (wrap_bytes > GPX_JSON_WRAP_BYTES || wrap_bytes <= GPX_JSON_WRAP_OVERHEAD + GPX_JSON_MAX_MEMBER)
    return fail(GPX_EINVAL, "wrap_bytes out of range");
  if (n_replies % E.S.L) return fail(GPX_EINVAL, "replies: n is not a multiple of n_lanes");
  if ((uint64_t)n_replies + n_dec_max + n_reqs > 0x7fffffffull) return fail(GPX_ERANGE, "too many records");
  const uint32_t nr = n_replies, nd = n_dec_max, nq = n_reqs, n = nr + nd + nq, L = E.S.L;
  if (n == 0) return GPX_OK;
  if ((rc = call.begin())) return rc;
  WireJsonEncArgs A;
  memset(&A, 0, sizeof A);
  A.R = encode_args(L, nr, nullptr, replies, rstatus_replies);
  A.D = encode_args(L, nd, n_dec_ptr, decisions, rstatus_decisions);
  A.Z = Z;
  A.n = n;
  A.L = L;
  A.T = (uint32_t)(wrap_bytes - GPX_JSON_WRAP_OVERHEAD - GPX_JSON_MAX_MEMBER);
  A.F.reqs = reqs;
  A.F.meta = meta;
  A.F.status = status;
  A.F.payload = payload;
  A.F.n = nq;
  A.F.n_down = n_down;
  A.F.rstatus = rstatus_reqs;
  /* scratch: the records' keys and stable orders, the member candidates, their sort and scans, the forwards' rows and
   * the down nodes */
  WireScan scan{json_enc_cub_bytes(ex, nr, nd, n)};
  uint32_t *iota, *rkey, *rperm, *rskey, *dkey, *dperm, *dskey, *order, *start, *off, *noff, *foff;
  int32_t* down;
  unsigned long long* skey;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
         iota = c.take<uint32_t>(n);
         rkey = c.take<uint32_t>(nr);
         rperm = c.take<uint32_t>(nr);
         rskey = c.take<uint32_t>(nr);
         dkey = c.take<uint32_t>(nd);
         dperm = c.take<uint32_t>(nd);
         dskey = c.take<uint32_t>(nd);
         A.first = c.take<uint32_t>((size_t)L * A.Z.n);
         A.mset = c.take<uint32_t>(n);
         A.mlane = c.take<uint8_t>(n);
         A.msize = c.take<uint32_t>(n);
         A.key = c.take<unsigned long long>(n);
         skey = c.take<unsigned long long>(n);
         order = c.take<uint32_t>(n);
         A.val = c.take<uint32_t>(n);
         start = c.take<uint32_t>(n);
         A.cnt = c.take<uint32_t>((size_t)JE_NCNT * n);
         off = c.take<uint32_t>((size_t)JE_NCNT * n);
         A.ncnt = c.take<uint32_t>(2ull * nr);
         noff = c.take<uint32_t>(2ull * nr);
         A.wbeg = c.take<uint2>(n);
         A.F.cnt = c.take<uint32_t>(2ull * nq);
         foff = c.take<uint32_t>(2ull * nq);
         A.fmem = c.take<uint8_t>(nq);
         A.flane = c.take<uint8_t>(nq);
         A.fdi = c.take<uint8_t>(nq);
         down = c.take<int32_t>(n_down);
         scan.lay(c, JE_NCNT + 4);
         return (size_t)0;
       })))
    return rc;
  if (nq && n_down && (rc = ex.upload(down, down_nodes, n_down * 4ull))) return rc;
  A.F.down = down;
  A.F.off = foff;
  A.R.key = rkey;
  A.R.perm = rperm;
  A.R.skey = rskey;
  A.D.key = dkey;
  A.D.perm = dperm;
  A.D.skey = dskey;
  A.skey = skey;
  A.order = order;
  A.start = start;
  A.off = off;
  A.noff = noff;
  if ((rc = ex.launch(k_wire_iota, n, 256, iota, n))) return rc;
  /* the byte encoders' classification and stable (lane, gid) / gid order */
  const WireAccArgs none{};
  for (int k = 0; k < 2; k++) {
    WireEncodeArgs& R = k ? A.D : A.R;
    if (R.n == 0) continue;
    if ((rc = wire_enc_launch(ex, E, k ? ENC_DECISIONS : ENC_REPLIES, true, R, none)) ||
        (rc = ex.sort((const uint32_t*)R.key, (uint32_t*)R.skey, iota, (uint32_t*)R.perm, R.n, 32, scan.cub,
                      scan.cub_bytes)))
      return rc;
  }
  if ((rc = ex.fill(A.first, 0xff, (size_t)L * A.Z.n * 4))) return rc;
  if (nr && (rc = ex.launch(k_json_enc_nacks, nr, 256, E.S, E.W, A))) return rc;
  if (nq && (rc = ex.launch(k_json_enc_fwd, nq, 128, E.S, E.W, A))) return rc;
  if ((rc = ex.launch(k_json_enc_members, n, 128, E.S, E.W, A)) || (rc = ex.launch(k_json_enc_keys, n, 256, A)) ||
      /* stable: the candidates are in sweep order, so members end up in (lane, first of their set, sweep) order */
      (rc = ex.sort((const unsigned long long*)A.key, skey, iota, order, n, 35, scan.cub, scan.cub_bytes)) ||
      (rc = ex.launch(k_json_enc_vals, n, 256, A)) || (rc = ex.sum_by_key(skey, A.val, start, n, scan)) ||
      (rc = ex.launch(k_json_enc_cut, n, 256, A)) || (rc = ex.scan(A.cnt, off, n, JE_NCNT, scan)) ||
      (rc = ex.totals(A.cnt, off, n, JE_NCNT, scan.tot)))
    return rc;
  if (nr) {
    if ((rc = ex.scan(A.ncnt, noff, nr, 2, scan)) || (rc = ex.totals(A.ncnt, noff, nr, 2, scan.tot + JE_NCNT)))
      return rc;
  } else if ((rc = ex.fill(scan.tot + JE_NCNT, 0, 8))) {
    return rc;
  }
  if (nq) {
    if ((rc = ex.scan(A.F.cnt, foff, nq, 2, scan)) || (rc = ex.totals(A.F.cnt, foff, nq, 2, scan.tot + JE_NCNT + 2)))
      return rc;
  } else if ((rc = ex.fill(scan.tot + JE_NCNT + 2, 0, 8))) {
    return rc;
  }
  uint32_t tot[JE_NCNT + 4];
  if ((rc = ex.read(tot, scan.tot, sizeof tot)) || (rc = ex.sync())) return rc; /* the one host read: the sizes */
  if (tot[JE_BIG]) return fail(GPX_EINVAL, "a member is larger than GPX_JSON_MAX_MEMBER");
  const uint64_t bytes = (uint64_t)tot[JE_BYTES] + tot[JE_NCNT] + tot[JE_NCNT + 2],
                 n_out = (uint64_t)tot[JE_REFS] + tot[JE_NCNT + 1] + tot[JE_NCNT + 3];
  if (bytes > 0xffffffffull || n_out > 0xffffffffull) return fail(GPX_ERANGE, "output larger than 4 GiB");
  const uint32_t sizes[2] = {(uint32_t)bytes, (uint32_t)n_out};
  if ((rc = wire_fit(o, sizes, "encode output too small"))) return rc;
  if (bytes == 0) return call.end();
  /* pass 1: the bare NACKs, the lone REQUEST packets, then the wrappers and their refs at the scanned offsets, left
   * in flight */
  A.nack_bytes = tot[JE_NCNT];
  A.n_nacks = tot[JE_NCNT + 1];
  A.lone_bytes = tot[JE_NCNT + 2];
  A.n_lone = tot[JE_NCNT + 3];
  A.out = out;
  A.refs = refs;
  if (A.n_nacks && (rc = ex.launch(k_json_enc_emit_nacks, nr, 128, E.S, E.W, A))) return rc;
  if (A.n_lone && (rc = ex.launch(k_json_enc_emit_fwd, nq, 128, E.S, E.W, A))) return rc;
  if ((rc = ex.launch(k_json_enc_emit, n, 128, E.S, E.W, A)) || (rc = ex.launch(k_json_enc_refs, n, 256, A)))
    return rc;
  return call.end();
}

/* ---- response cache (gpx_respcache.cuh) ------------------------------------------------------------------------------ */
/* gpx_response_cache_put_device; T is the engine's table */
template <class Ex, class C>
static int rc_put(Ex& ex, C& call, void** buf, size_t* buf_bytes, const RcTable& T, uint32_t n,
                  const gpx_rc_key* keys, int64_t now_ms) {
  if (n && !keys) return fail(GPX_EINVAL, "null argument");
  if (n == 0) return GPX_OK;
  int rc = call.begin();
  if (rc) return rc;
  RcPutArgs A;
  memset(&A, 0, sizeof A);
  A.keys = keys;
  A.n = n;
  A.now_ms = now_ms;
  GidSort sort(ex, n, T.mask); /* the bucket's key bits */
  if ((rc = wire_place(ex, buf, buf_bytes, [&](Carve& c) {
         A.bucket = c.take<uint32_t>(n);
         A.gen = c.take<uint32_t>(n);
         A.bad = c.take<uint32_t>(1);
         sort.lay(c);
         return (size_t)0;
       })))
    return rc;
  uint32_t bad = 0;
  if ((rc = ex.fill(A.bad, 0, 4)) || (rc = ex.launch(k_rc_put_keys, n, 256, T, A)) || (rc = ex.read(&bad, A.bad, 4)) ||
      (rc = ex.sync())) /* the one host read: a bad key writes nothing */
    return rc;
  if (bad) return fail(GPX_EINVAL, "response cache: a key with a negative handle or gid >= max_groups");
  if ((rc = sort.run(ex, A.bucket, n))) return rc;
  A.perm = sort.perm;
  A.sbucket = sort.skeys;
  if ((rc = ex.launch(k_rc_put, n, 256, T, A))) return rc;
  return call.end();
}

/* gpx_response_cache_match_device */
template <class Ex, class C>
static int rc_match(Ex& ex, C& call, void** buf, size_t* buf_bytes, const RcTable& T, uint32_t n,
                    const gpx_request_rec* reqs, const gpx_wire_req_meta* meta, int64_t now_ms, int32_t* hit,
                    gpx_request_rec* out_reqs, gpx_wire_req_meta* out_meta, uint32_t* n_out) {
  if (!n_out || (n && (!reqs || !meta || !hit || !out_reqs || !out_meta))) return fail(GPX_EINVAL, "null argument");
  *n_out = 0;
  if (n == 0) return GPX_OK;
  int rc = call.begin();
  if (rc) return rc;
  RcMatchArgs A;
  memset(&A, 0, sizeof A);
  A.reqs = reqs;
  A.meta = meta;
  A.n = n;
  A.now_ms = now_ms;
  A.hit = hit;
  A.out_reqs = out_reqs;
  A.out_meta = out_meta;
  GidSort sort(ex, n, 0xffffffffu); /* all 32 bits of the client values */
  WireScan scan{wire_cub_bytes(ex, n, 32)};
  uint32_t* client;
  uint32_t* off;
  if ((rc = wire_place(ex, buf, buf_bytes, [&](Carve& c) {
         client = c.take<uint32_t>(n);
         A.dup = c.take<uint32_t>(n);
         A.miss = c.take<uint32_t>(n);
         off = c.take<uint32_t>(n);
         scan.lay(c, 1);
         sort.lay(c);
         return (size_t)0;
       })))
    return rc;
  A.off = off;
  /* the client values out of the 32-byte records (the last word), sorted */
  if ((rc = ex.column(client, &reqs->client, sizeof(gpx_request_rec), n)) || (rc = sort.run(ex, client, n))) return rc;
  A.perm = sort.perm;
  A.sclient = sort.skeys;
  uint32_t tot = 0;
  if ((rc = ex.launch(k_rc_dups, n, 256, A)) || (rc = ex.launch(k_rc_match, n, 256, T, A)) ||
      (rc = wire_scan(ex, A.miss, off, n, 1, scan, &tot)) || (rc = ex.launch(k_rc_scatter, n, 256, A)) ||
      (rc = ex.sync())) /* the one host read: the count of misses */
    return rc;
  *n_out = tot;
  return call.end();
}

/* ---- journal frames (gpx_journal.cuh) --------------------------------------------------------------------------------
 * gpx_log_frame_device over [*from, head), head being the engine's head of the lane.  Before the one synchronisation
 * only the range is known on the host, so the directory and the counters are sized from it: an image takes at least 32
 * ring bytes and a segment at least GPX_SEG_DEC_BYTES(1). */
template <class Ex, class C>
static int log_frame(Ex& ex, C& call, const WireEnv& E, uint32_t lane, uint64_t* from, uint64_t head,
                     const gpx_journal_req* meta, uint32_t n_meta, uint8_t* out, uint64_t* out_bytes,
                     uint32_t* n_frames, gpx_journal_miss* missing, uint32_t* n_missing) {
  WireOut o[] = {{out_bytes, out != nullptr}, {n_frames, out != nullptr}, {n_missing, missing != nullptr}};
  int rc = wire_args(from && (!n_meta || meta), 0, o);
  if (rc) return rc;
  if (*from & 31) return fail(GPX_EINVAL, "from is not a segment boundary");
  if (*from > head) return fail(GPX_EINVAL, "from is beyond the head");
  if (*from == head) return GPX_OK;
  const uint64_t range = head - *from;
  if (range > E.S.ring_cap) return fail(GPX_ERANGE, "bytes from `from` on were already overwritten");
  if (range / 32 > 0xffffffffull) return fail(GPX_ERANGE, "range too long for one call");
  if ((rc = call.begin())) return rc;
  const uint32_t n = (uint32_t)(range / 32);
  const uint32_t seg_cap = (uint32_t)std::min<uint64_t>(range / GPX_SEG_DEC_BYTES(1) + 2, 1ull << 20);
  WireScan scan{ex.scan_bytes(n)};
  JournalArgs A;
  memset(&A, 0, sizeof A);
  A.lane = lane;
  A.n = n;
  A.meta = meta;
  A.n_meta = n_meta;
  LogSeg* segs;
  unsigned long long* ctl;
  uint32_t* off;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
         segs = c.take<LogSeg>(seg_cap);
         ctl = c.take<unsigned long long>(JF_NCTL);
         A.cnt = c.take<uint32_t>((size_t)JF_NCNT * n);
         off = c.take<uint32_t>((size_t)JF_NCNT * n);
         scan.lay(c, JF_NCNT);
         return (size_t)0;
       })))
    return rc;
  A.segs = segs;
  A.ctl = ctl;
  LogFindArgs D;
  memset(&D, 0, sizeof D);
  D.lane = lane;
  D.from = *from;
  D.segs = segs;
  D.seg_cap = seg_cap;
  D.ctl = ctl;
  /* pass 0: the directory, the table's order, each image's frame bytes, frame and misses, their scans */
  if ((rc = ex.fill(ctl, 0, JF_NCTL * sizeof(unsigned long long))) || (rc = ex.launch(k_log_dir, 1, 32, E.S, D)) ||
      (n_meta && (rc = ex.launch(k_journal_meta, n_meta, 256, A))) ||
      (rc = ex.launch(k_journal, n, GPX_JOURNAL_BLOCK, E.S, E.W, A)) || (rc = ex.scan(A.cnt, off, n, JF_NCNT, scan)) ||
      (rc = ex.totals(A.cnt, off, n, JF_NCNT, scan.tot)))
    return rc;
  A.off = off;
  uint32_t tot[JF_NCNT];
  unsigned long long c[JF_NCTL];
  if ((rc = ex.launch(k_journal_fit, n, 256, A)) || (rc = ex.read(tot, scan.tot, sizeof tot)) ||
      (rc = ex.read(c, ctl, sizeof c)) || (rc = ex.sync())) /* the one host read: the sizes and the flags */
    return rc;
  if (c[LOGF_ERR] == LOGF_OVERWRITTEN) return fail(GPX_ERANGE, "bytes from `from` on were already overwritten");
  if (c[LOGF_ERR] == LOGF_CORRUPT) return fail(GPX_EINVAL, "`from` is not a segment boundary");
  if (c[LOGF_ERR] == LOGF_TOO_MANY) return fail(GPX_ERANGE, "more log segments than the directory holds");
  if (c[LOGF_HEAD] != head) return fail(GPX_EINVAL, "the head moved: order the calls that log before this one");
  if (c[JF_UNSORTED]) return fail(GPX_EINVAL, "meta is not strictly ascending by (gid, req_id)");
  if (c[JF_BAD_BLOB]) return fail(GPX_EINVAL, "an ACCEPT image's request blob lies outside its segment");
  if (tot[JF_MISS]) { /* the misses, and no frame */
    const uint32_t sizes[3] = {0, 0, tot[JF_MISS]};
    if ((rc = wire_fit(o, sizes, "missing too small"))) return rc;
    A.miss = missing;
    A.emit = 1;
    if ((rc = ex.launch(k_journal, n, GPX_JOURNAL_BLOCK, E.S, E.W, A)) || (rc = call.end())) return rc;
    return fail(GPX_ENOENT, "requests or names the frames need are missing");
  }
  if (c[JF_OVER]) return fail(GPX_ERANGE, "the frames pass 4 GiB");
  const uint32_t sizes[3] = {tot[JF_BYTES], tot[JF_FRAMES], 0};
  if ((rc = wire_fit(o, sizes, "frame output too small"))) return rc;
  if (tot[JF_FRAMES]) { /* pass 1: the frames at the scanned offsets, left in flight */
    A.out = out;
    A.emit = 2;
    if ((rc = ex.launch(k_journal, n, GPX_JOURNAL_BLOCK, E.S, E.W, A))) return rc;
  }
  *from = head;
  return call.end();
}

/* ---- journal garbage collection (gpx_journal_gc.cuh) -----------------------------------------------------------------
 * gpx_journal_compact_device.  Everything up to the one synchronisation is enqueued without a host read, malformed
 * frames included (they are neither indexed nor kept), so that the totals of the counters, the bad count and the
 * flag on file_off come back together. */
template <class Ex, class C>
static int journal_compact(Ex& ex, C& call, const WireEnv& E, const uint8_t* bytes, uint64_t n_bytes,
                           const uint32_t* file_off, uint32_t n_files, const uint32_t* starts, uint32_t n,
                           const int32_t* gc_slot, uint32_t n_gids, uint32_t last_readonly, uint8_t* out,
                           uint64_t* out_bytes, gpx_journal_file* files, uint32_t* bad, uint32_t* n_bad) {
  WireOut o[] = {{out_bytes, out != nullptr}, {n_bad, bad != nullptr}};
  int rc = wire_args((!n_bytes || bytes) && (!n || starts) && (!n_files || (file_off && files && gc_slot)), n_bytes, o);
  if (rc) return rc;
  if (n_files == 0) return n ? fail(GPX_EINVAL, "frames without a file") : GPX_OK;
  if (n_gids < E.S.G) return fail(GPX_EINVAL, "gc_slot needs one slot per group (n_gids < max_groups)");
  if ((rc = call.begin())) return rc;
  JournalGcArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.n_bytes = (uint32_t)n_bytes;
  A.file_off = file_off;
  A.n_files = n_files;
  A.starts = starts;
  A.n = n;
  A.gc_slot = gc_slot;
  A.last_readonly = last_readonly;
  GidSort sort(ex, n, E.S.G); /* key G: not indexed */
  WireScan scan{ex.scan_bytes(n)}, fscan{ex.scan_bytes(n_files)};
  uint32_t *cnt, *off, *foff;
  if ((rc = wire_place(ex, E.buf, E.bytes, [&](Carve& c) {
         A.bad_off = c.take<uint32_t>(1);
         A.rec = c.take<JgcRec>(n);
         A.key = c.take<uint32_t>(n);
         cnt = c.take<uint32_t>((size_t)JG_NCNT * n);
         off = c.take<uint32_t>((size_t)JG_NCNT * n);
         scan.lay(c, JG_NCNT);
         sort.lay(c);
         A.fs = c.take<JgcFile>(n_files);
         A.fbytes = c.take<uint32_t>(n_files);
         foff = c.take<uint32_t>(n_files);
         fscan.lay(c, 1);
         return (size_t)0;
       })))
    return rc;
  A.cnt = cnt;
  A.off = off;
  A.tot = scan.tot;
  A.foff = foff;
  /* parse, sort the indexed frames by gid, keep, scan; then the files and the scan of their compacted bytes */
  if ((rc = ex.fill(A.bad_off, 0, 4)) || (rc = ex.launch(k_jgc_offsets, n_files + 1, 256, A))) return rc;
  if (n) {
    if ((rc = ex.launch(k_jgc_parse, n, 128, E.S, E.W, A)) || (rc = sort.run(ex, A.key, n))) return rc;
    A.perm = sort.perm;
    A.skey = sort.skeys;
    if ((rc = ex.launch(k_jgc_keep, n, 256, A)) || (rc = ex.scan(cnt, off, n, JG_NCNT, scan)) ||
        (rc = ex.totals(cnt, off, n, JG_NCNT, scan.tot)))
      return rc;
  } else if ((rc = ex.fill(scan.tot, 0, JG_NCNT * sizeof(uint32_t)))) {
    return rc;
  }
  uint32_t tot[JG_NCNT], ftot = 0, bad_off = 0;
  if ((rc = ex.launch(k_jgc_file, n_files, 128, A)) || (rc = ex.scan(A.fbytes, foff, n_files, 1, fscan)) ||
      (rc = ex.totals(A.fbytes, foff, n_files, 1, fscan.tot)) || (rc = ex.read(tot, scan.tot, sizeof tot)) ||
      (rc = ex.read(&ftot, fscan.tot, 4)) || (rc = ex.read(&bad_off, A.bad_off, 4)) ||
      (rc = ex.sync())) /* the one host read: the totals and the flag */
    return rc;
  if (bad_off) return fail(GPX_EINVAL, "file_off is not ascending from 0 to n_bytes");
  if (tot[JG_BAD]) { /* the malformed frames' indices, and nothing else */
    const uint32_t sizes[2] = {0, tot[JG_BAD]};
    if ((rc = wire_fit(o, sizes, "bad too small"))) return rc;
    A.bad = bad;
    if ((rc = ex.launch(k_jgc_bad, n, 256, A)) || (rc = call.end())) return rc;
    return fail(GPX_EINVAL, "frames that do not parse or do not chain");
  }
  const uint32_t sizes[2] = {ftot, 0};
  if ((rc = wire_fit(o, sizes, "out too small"))) return rc;
  A.out = out;
  A.files = files;
  if (ftot && (rc = ex.launch(k_jgc_copy, (uint32_t)std::min<uint64_t>((uint64_t)n * 32u, 32ull * GPX_JGC_COPY_WARPS),
                              256, A)))
    return rc;
  if ((rc = ex.launch(k_jgc_files, n_files, 128, A))) return rc;
  return call.end();
}

/* gpx_journal_index's walk (journal.read_journal's) */
static int journal_index(const uint8_t* buf, uint64_t n_bytes, uint32_t base, uint32_t* starts, uint32_t cap,
                         uint32_t* n_frames, uint64_t* end) {
  if (!n_frames || !end || (n_bytes && !buf) || (cap && !starts)) return fail(GPX_EINVAL, "null argument");
  if (base + n_bytes > 0xffffffffull) return fail(GPX_EINVAL, "base + n_bytes passes 4 GiB");
  uint64_t p = 0;
  uint32_t k = 0;
  while (p + 4 <= n_bytes) {
    const uint32_t l = ((uint32_t)buf[p] << 24) | ((uint32_t)buf[p + 1] << 16) | ((uint32_t)buf[p + 2] << 8) | buf[p + 3];
    if (l >= 0x80000000u || p + 4 + l > n_bytes) break; /* torn tail */
    if (k < cap) starts[k] = base + (uint32_t)p;
    k++;
    p += 4 + l;
  }
  *n_frames = k;
  *end = p;
  return k > cap ? fail(GPX_ERANGE, "more frames than cap") : GPX_OK;
}
