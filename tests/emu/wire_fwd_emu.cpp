/*
 * wire_fwd_emu.cpp -- k_wire_fwd and k_json_req (gigapaxos_b200/csrc/gpx_wire_fwd.cuh, the source the GPU runs)
 * compiled for the host over cuda_emu.h, beside the byte and JSON decoders of wire_json_emu.cpp (same engine state).
 * The acceptor and coordinator rows the routing reads, and the batching settings, are set from the test.  The scans
 * and the stable sort by gid that gpx_wire_host.inc does with CUB are done here with the standard library.  Test
 * infrastructure only.
 */
#include "wire_json_emu.cpp"

#include "gpx_wire_fwd.cuh"

/* live groups gids[0..n) with one member set m[0..R) (sorted ascending), interned once as gpx_create_groups interns
 * it: worlds of more groups than there are member-set slots */
extern "C" int emu_wire_groups_alike(void* p, uint32_t n, const uint32_t* gids, uint32_t R, const int32_t* m) {
  EmuWire* x = static_cast<EmuWire*>(p);
  if (n == 0) return 0;
  if (emu_wire_group(p, gids[0], R, m)) return -1;
  for (uint32_t k = 1; k < n; k++) {
    if (gids[k] >= x->S.G) return -1;
    x->meta[gids[k]] = x->meta[gids[0]];
  }
  return 0;
}

/* the rows propose_route reads, [L][G] each (the caller keeps them alive), and RequestBatcher's settings */
extern "C" void emu_fwd_state(void* p, int4* acc_row, uint32_t* acc_aux, int4* coord_row, int32_t batching,
                              int32_t max_batch_size, int32_t size_est, long long max_batch_bytes) {
  EmuWire* x = static_cast<EmuWire*>(p);
  x->S.acc_row = acc_row;
  x->S.acc_aux = acc_aux;
  x->S.coord_row = coord_row;
  x->S.batching = batching;
  x->S.max_batch_size = max_batch_size;
  x->S.size_est = size_est;
  x->S.max_batch_bytes = max_batch_bytes;
}

/* gpx_wire_encode_forwards_device without the copies; sizes[2] = {bytes, refs} in / out, GPX_ERANGE when too small */
extern "C" int emu_wire_encode_forwards(void* p, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta, uint32_t n,
                                        const int32_t* status, const uint8_t* payload, uint32_t n_down,
                                        const int32_t* down, uint8_t* rstatus, uint8_t* out, gpx_wire_ref* refs,
                                        uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  std::vector<uint32_t> cnt(2 * (size_t)n + 1), off(2 * (size_t)n + 1);
  WireFwdArgs A;
  memset(&A, 0, sizeof A);
  A.reqs = reqs;
  A.meta = meta;
  A.status = status;
  A.payload = payload;
  A.down = down;
  A.n = n;
  A.n_down = n_down;
  A.rstatus = rstatus;
  A.cnt = cnt.data();
  A.off = off.data();
  emu_launch(k_wire_fwd, (n + block - 1) / block, block, x->S, x->W, A);
  uint64_t tot[2];
  exclusive_rows(cnt, off, n, 2, tot);
  const bool small = tot[0] > sizes[0] || tot[1] > sizes[1];
  sizes[0] = tot[0];
  sizes[1] = tot[1];
  if (small) return GPX_ERANGE;
  A.out = out;
  A.refs = refs;
  A.emit = 1;
  emu_launch(k_wire_fwd, (n + block - 1) / block, block, x->S, x->W, A);
  return 0;
}

/* gpx_wire_decode_json_requests_device without the copies; sizes[2] = {requests, payload bytes} in / out */
extern "C" int emu_wire_decode_json_requests(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                             const gpx_wire_ref* pkts, uint32_t n_pkts, const gpx_wire_member* mem,
                                             int64_t now_ms, int32_t* status, gpx_request_rec* reqs,
                                             gpx_wire_req_meta* meta, uint8_t* payload, uint64_t* sizes,
                                             uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  std::vector<uint32_t> cnt((size_t)WQ_NCNT * n + 1), off((size_t)WQ_NCNT * n + 1);
  WireJsonReqArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.mem = mem;
  A.n_bytes = n_bytes;
  A.n_pkts = n_pkts;
  A.n = n;
  A.now_ms = now_ms;
  A.status = status;
  A.cnt = cnt.data();
  A.off = off.data();
  emu_launch(k_json_req, (n + block - 1) / block, block, x->S, x->W, A);
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
  emu_launch(k_json_req, (n + block - 1) / block, block, x->S, x->W, A);
  const std::vector<uint32_t> perm = stable_order(key);
  gather(perm, sq, reqs);
  gather(perm, sm, meta);
  return 0;
}
