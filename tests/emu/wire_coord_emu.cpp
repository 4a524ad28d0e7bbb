/*
 * wire_coord_emu.cpp -- the coordinator's wire kernels (k_wire_req_decode, k_wire_enc_keys_accepts and
 * k_wire_enc_accepts, gigapaxos_b200/csrc/gpx_wire_dev.cuh) compiled for the host over cuda_emu.h.  The engine, group
 * and name set-up of wire_emu.cpp is reused as it is; the scans and the stable sorts by gid are done with the standard
 * library.  Test infrastructure only.
 */
#include "wire_emu.cpp"

/* gpx_wire_decode_requests_device without the copies; sizes[2] = {requests, payload bytes} in / out; GPX_ERANGE when
 * an output is too small (nothing but status written then) */
extern "C" int emu_wire_decode_requests(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                        const gpx_wire_ref* pkts, int64_t now_ms, int32_t* status,
                                        gpx_request_rec* reqs, gpx_wire_req_meta* meta, uint8_t* payload,
                                        uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  std::vector<uint32_t> cnt((size_t)WQ_NCNT * n + 1), off((size_t)WQ_NCNT * n + 1);
  WireReqDecodeArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.n_bytes = n_bytes;
  A.n = n;
  A.now_ms = now_ms;
  A.cnt = cnt.data();
  A.off = off.data();
  A.status = status;
  emu_launch(k_wire_req_decode, (n + block - 1) / block, block, x->S, x->W, A);
  uint64_t tot[WQ_NCNT];
  exclusive_rows(cnt, off, n, WQ_NCNT, tot);
  const bool small = tot[WQ_REQ] > sizes[0] || tot[WQ_PAY] > sizes[1];
  sizes[0] = tot[WQ_REQ];
  sizes[1] = tot[WQ_PAY];
  if (small) return GPX_ERANGE;
  const size_t nq = tot[WQ_REQ];
  std::vector<gpx_request_rec> sq(nq + 1);
  std::vector<gpx_wire_req_meta> sm(nq + 1);
  std::vector<uint32_t> key(nq);
  A.req = sq.data();
  A.meta = sm.data();
  A.key = key.data();
  A.payload = payload;
  A.emit = 1;
  emu_launch(k_wire_req_decode, (n + block - 1) / block, block, x->S, x->W, A);
  std::vector<uint32_t> perm = stable_order(key);
  for (size_t i = 0; i < nq; i++) {
    reqs[i] = sq[perm[i]];
    meta[i] = sm[perm[i]];
  }
  return 0;
}

/* gpx_wire_encode_accepts_device without the copies: the keys, the sort and the passes run over n_max ACCEPTs, their
 * count read from *n_ptr as the device reads it.  sizes[2] = {bytes, refs} in / out. */
extern "C" int emu_wire_encode_accepts(void* p, const uint32_t* n_ptr, uint32_t n_max, const gpx_accept_rec* recs,
                                       const uint32_t* heads, const gpx_request_rec* reqs,
                                       const gpx_wire_req_meta* meta, uint32_t n_reqs, const uint8_t* payload,
                                       uint8_t* rstatus, uint8_t* out, gpx_wire_ref* refs, uint64_t* sizes,
                                       uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  const uint32_t n = n_max;
  std::vector<uint32_t> key(n + 1), perm, skey(n + 1), cnt(2 * (size_t)n + 1), off(2 * (size_t)n + 1);
  WireEncodeArgs A;
  memset(&A, 0, sizeof A);
  A.recs = recs;
  A.n = n;
  A.n_lanes = x->S.L;
  A.rstatus = rstatus;
  A.key = key.data();
  A.n_ptr = n_ptr;
  WireAccArgs X;
  X.head = heads;
  X.reqs = reqs;
  X.meta = meta;
  X.n_reqs = n_reqs;
  X.payload = payload;
  emu_launch(k_wire_enc_keys_accepts, (n + block - 1) / block, block, x->S, x->W, A, X);
  key.resize(n);
  perm = stable_order(key);
  for (uint32_t i = 0; i < n; i++) skey[i] = key[perm[i]];
  A.perm = perm.data();
  A.skey = skey.data();
  A.cnt = cnt.data();
  A.off = off.data();
  emu_launch(k_wire_enc_accepts, (n + block - 1) / block, block, x->S, x->W, A, X);
  uint64_t tot[2];
  exclusive_rows(cnt, off, n, 2, tot);
  const bool small = tot[0] > sizes[0] || tot[1] > sizes[1];
  sizes[0] = tot[0];
  sizes[1] = tot[1];
  if (small) return GPX_ERANGE;
  A.out = out;
  A.refs = refs;
  A.emit = 1;
  emu_launch(k_wire_enc_accepts, (n + block - 1) / block, block, x->S, x->W, A, X);
  return 0;
}
