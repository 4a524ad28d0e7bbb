/*
 * wire_json_sweep_emu.cpp -- gpx_wire_encode_json_sweep_device's kernels (gigapaxos_b200/csrc/gpx_wire_json_enc.cuh
 * and the forwarding walk of gpx_wire_fwd.cuh, the source the GPU runs) compiled for the host over cuda_emu.h, on top
 * of the JSON-out emulator (wire_json_out_emu.cpp, whose emu_wire_encode_json is the no-forwards call to compare
 * with).  The stable radix sorts, the scans and the scan by key that gpx_wire_host.inc does with CUB are done here with
 * the standard library.  Test infrastructure only.
 */
#include "wire_json_out_emu.cpp"

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

/* gpx_wire_encode_json_sweep_device without the copies: sizes[2] = {bytes, refs} capacities in, sizes out.  Returns 0,
 * -5 (GPX_ERANGE: sizes reported, no packet written) or -1 (GPX_EINVAL: wrap_bytes out of range, an oversized reply or
 * commit member). */
extern "C" int emu_wire_encode_json_sweep(void* p, uint32_t nr, const gpx_accept_reply_rec* rep,
                                          const gpx_decision_rec* dec, const uint32_t* n_dec_ptr, uint32_t nd,
                                          const gpx_request_rec* reqs, const gpx_wire_req_meta* meta, uint32_t nq,
                                          const int32_t* status, const uint8_t* payload, uint32_t n_down,
                                          const int32_t* down, uint8_t* rst_r, uint8_t* rst_d, uint8_t* rst_q,
                                          uint64_t wrap_bytes, uint8_t* out, gpx_wire_ref* refs, uint64_t* sizes,
                                          uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  if (wrap_bytes == 0) wrap_bytes = GPX_JSON_WRAP_BYTES;
  if (wrap_bytes > GPX_JSON_WRAP_BYTES || wrap_bytes <= GPX_JSON_WRAP_OVERHEAD + GPX_JSON_MAX_MEMBER) return GPX_EINVAL;
  const uint32_t n = nr + nd + nq, L = x->S.L;
  if (n == 0) {
    sizes[0] = sizes[1] = 0;
    return 0;
  }
  JsonSetTable T;
  T.grow(x->msets.data(), x->msets.size());
  std::vector<uint32_t> rkey(nr + 1), rperm, rskey(nr + 1), dkey(nd + 1), dperm, dskey(nd + 1),
      first((size_t)L * T.count.size(), GPX_JSON_ENC_NONE), mset(n), msize(n), order, val(n), start(n),
      cnt((size_t)JE_NCNT * n), off((size_t)JE_NCNT * n), ncnt(2ull * nr + 1), noff(2ull * nr + 1),
      fcnt(2ull * nq + 1), foff(2ull * nq + 1);
  std::vector<uint8_t> mlane(n), fmem(nq + 1), flane(nq + 1), fdi(nq + 1);
  std::vector<unsigned long long> key(n), skey(n);
  std::vector<uint2> wbeg(n);
  WireJsonEncArgs A;
  memset(&A, 0, sizeof A);
  for (int k = 0; k < 2; k++) {
    WireEncodeArgs& X = k ? A.D : A.R;
    X.recs = k ? (const void*)dec : (const void*)rep;
    X.n = k ? nd : nr;
    X.n_lanes = L;
    X.rstatus = k ? rst_d : rst_r;
    X.n_ptr = k ? n_dec_ptr : nullptr;
    X.key = (k ? dkey : rkey).data();
  }
  A.Z = {T.of_mset.data(), T.one.data(), T.nodes.data(), T.count.data(), (uint32_t)T.count.size()};
  A.n = n;
  A.L = L;
  A.T = (uint32_t)(wrap_bytes - GPX_JSON_WRAP_OVERHEAD - GPX_JSON_MAX_MEMBER);
  A.first = first.data();
  A.mset = mset.data();
  A.mlane = mlane.data();
  A.msize = msize.data();
  A.key = key.data();
  A.val = val.data();
  A.cnt = cnt.data();
  A.ncnt = ncnt.data();
  A.wbeg = wbeg.data();
  A.F.reqs = reqs;
  A.F.meta = meta;
  A.F.status = status;
  A.F.payload = payload;
  A.F.down = down;
  A.F.n = nq;
  A.F.n_down = n_down;
  A.F.rstatus = rst_q;
  A.F.cnt = fcnt.data();
  A.fmem = fmem.data();
  A.flane = flane.data();
  A.fdi = fdi.data();
  const auto grid = [&](uint32_t k) { return (k + block - 1) / block; };
  /* the byte encoders' keys and stable sorts */
  if (nr) {
    emu_launch(k_wire_enc_keys_replies, grid(nr), block, x->S, x->W, A.R);
    rkey.resize(nr);
    rperm = stable_order(rkey);
    for (uint32_t i = 0; i < nr; i++) rskey[i] = rkey[rperm[i]];
    A.R.perm = rperm.data();
    A.R.skey = rskey.data();
  }
  if (nd) {
    emu_launch(k_wire_enc_keys_decisions, grid(nd), block, x->S, x->W, A.D);
    dkey.resize(nd);
    dperm = stable_order(dkey);
    for (uint32_t i = 0; i < nd; i++) dskey[i] = dkey[dperm[i]];
    A.D.perm = dperm.data();
    A.D.skey = dskey.data();
  }
  if (nr) emu_launch(k_json_enc_nacks, grid(nr), block, x->S, x->W, A);
  if (nq) emu_launch(k_json_enc_fwd, grid(nq), block, x->S, x->W, A);
  emu_launch(k_json_enc_members, grid(n), block, x->S, x->W, A);
  emu_launch(k_json_enc_keys, grid(n), block, A);
  order.resize(n);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  for (uint32_t j = 0; j < n; j++) skey[j] = key[order[j]];
  A.skey = skey.data();
  A.order = order.data();
  emu_launch(k_json_enc_vals, grid(n), block, A);
  for (uint32_t j = 0, s = 0; j < n; j++) { /* exclusive sum by key */
    if (j == 0 || skey[j] != skey[j - 1]) s = 0;
    start[j] = s;
    s += val[j];
  }
  A.start = start.data();
  emu_launch(k_json_enc_cut, grid(n), block, A);
  uint64_t tot[JE_NCNT], ntot[2] = {0, 0}, ftot[2] = {0, 0};
  exclusive_rows(cnt, off, n, JE_NCNT, tot);
  if (nr) exclusive_rows(ncnt, noff, nr, 2, ntot);
  if (nq) exclusive_rows(fcnt, foff, nq, 2, ftot);
  A.off = off.data();
  A.noff = noff.data();
  A.F.off = foff.data();
  if (tot[JE_BIG]) return GPX_EINVAL;
  const uint64_t bytes = tot[JE_BYTES] + ntot[0] + ftot[0], n_refs = tot[JE_REFS] + ntot[1] + ftot[1];
  const bool small = bytes > sizes[0] || n_refs > sizes[1];
  sizes[0] = bytes;
  sizes[1] = n_refs;
  if (small) return GPX_ERANGE;
  A.nack_bytes = (uint32_t)ntot[0];
  A.n_nacks = (uint32_t)ntot[1];
  A.lone_bytes = (uint32_t)ftot[0];
  A.n_lone = (uint32_t)ftot[1];
  A.out = out;
  A.refs = refs;
  if (A.n_nacks) emu_launch(k_json_enc_emit_nacks, grid(nr), block, x->S, x->W, A);
  if (A.n_lone) emu_launch(k_json_enc_emit_fwd, grid(nq), block, x->S, x->W, A);
  emu_launch(k_json_enc_emit, grid(n), block, x->S, x->W, A);
  emu_launch(k_json_enc_refs, grid(n), block, A);
  return 0;
}
