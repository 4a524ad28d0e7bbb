/*
 * wire_device_emu.cpp -- the decisions encoder of gpx_wire_encode_decisions_device (k_wire_enc_keys_decisions and
 * k_wire_enc_decisions with WireEncodeArgs.n_ptr, gigapaxos_b200/csrc/gpx_wire_dev.cuh) compiled for the host over
 * cuda_emu.h.  The engine, group and name set-up of wire_emu.cpp is reused as it is.  Test infrastructure only.
 */
#include "wire_emu.cpp"

/* gpx_wire_encode_decisions_device without the copies: the keys, the sort and the passes run over n_max records, the
 * record count is read from *n_ptr as the device reads it.  sizes[2] = {bytes, refs} in / out. */
extern "C" int emu_wire_encode_decisions_n(void* p, const uint32_t* n_ptr, uint32_t n_max, const void* recs,
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
  emu_launch(k_wire_enc_keys_decisions, (n + block - 1) / block, block, x->S, x->W, A);
  key.resize(n);
  perm = stable_order(key);
  for (uint32_t i = 0; i < n; i++) skey[i] = key[perm[i]];
  A.perm = perm.data();
  A.skey = skey.data();
  A.cnt = cnt.data();
  A.off = off.data();
  emu_launch(k_wire_enc_decisions, (n + block - 1) / block, block, x->S, x->W, A);
  uint64_t tot[2];
  exclusive_rows(cnt, off, n, 2, tot);
  const bool small = tot[0] > sizes[0] || tot[1] > sizes[1];
  sizes[0] = tot[0];
  sizes[1] = tot[1];
  if (small) return GPX_ERANGE;
  A.out = out;
  A.refs = refs;
  A.emit = 1;
  emu_launch(k_wire_enc_decisions, (n + block - 1) / block, block, x->S, x->W, A);
  return 0;
}
