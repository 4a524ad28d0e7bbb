/*
 * wire_json_emu.cpp -- the kernels of gigapaxos_b200/csrc/gpx_wire_json.cuh (the source the GPU runs) compiled for the
 * host over cuda_emu.h, beside the byte decoder of wire_emu.cpp (same engine state, so one world serves both).  Build
 * with -DGPX_JSON_CHUNK=<bytes> to cut packets into chunks that small.  The scans, the scan by packet and the stable
 * sorts by gid that gpx_wire_host.inc does with CUB are done here with the standard library.  Test infrastructure only.
 */
#include "wire_emu.cpp"

#include "gpx_wire_json.cuh"

/* gpx_wire_decode_json_device without the copies; sizes[3] = {members, replies, decisions} capacities in, sizes out;
 * returns -5 (GPX_ERANGE) when an output is too small, -1 (GPX_EINVAL) when the lengths exceed the arena */
extern "C" int emu_wire_decode_json(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                    const gpx_wire_ref* pkts, int32_t* status, gpx_wire_member* members,
                                    gpx_accept_reply_rec* rep, gpx_decision_rec* dec, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  if (n == 0) {
    sizes[0] = sizes[1] = sizes[2] = 0;
    return 0;
  }
  const uint32_t cap_items = (uint32_t)(n_bytes / GPX_JSON_CHUNK + 2ull * n + 1ull);
  const uint32_t cap_ev = (uint32_t)((uint64_t)cap_items * GPX_JSON_CHUNK / 2 + n + 1);
  const uint32_t cap_mem = (uint32_t)((uint64_t)cap_items * GPX_JSON_CHUNK / GPX_JSON_MIN_MEMBER + n + 1);
  std::vector<uint32_t> pcnt(2 * (size_t)n), poff(2 * (size_t)n), bad(n), pp(3 * (size_t)n), ikey(cap_items),
      ecnt(2 * (size_t)cap_items), eoff(2 * (size_t)cap_items), ev_open(cap_ev), ev_close(cap_ev),
      mcnt(3 * (size_t)cap_mem), moff(3 * (size_t)cap_mem);
  std::vector<JsonSum> isum(cap_items), ipre(cap_items);
  std::vector<gpx_wire_member> mem(cap_mem);
  WireJsonArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.n_bytes = n_bytes;
  A.n = n;
  A.status = status;
  A.pcnt = pcnt.data();
  A.poff = poff.data();
  A.bad = bad.data();
  A.pp = pp.data();
  A.cap_items = cap_items;
  A.ikey = ikey.data();
  A.isum = isum.data();
  A.ipre = ipre.data();
  A.ecnt = ecnt.data();
  A.eoff = eoff.data();
  A.ev_open = ev_open.data();
  A.ev_close = ev_close.data();
  A.cap_mem = cap_mem;
  A.mem = mem.data();
  A.mcnt = mcnt.data();
  A.moff = moff.data();
  const auto grid = [&](uint32_t k) { return (k + block - 1) / block; };
  uint64_t tot[3];
  emu_launch(k_json_pre, grid(n), block, A);
  exclusive_rows(pcnt, poff, n, 1, tot);
  emu_launch(k_json_sum, grid(cap_items), block, A);
  { /* exclusive scan by key */
    JsonSum acc = json_identity();
    for (uint32_t i = 0; i < cap_items; i++) {
      if (i == 0 || ikey[i] != ikey[i - 1]) acc = json_identity();
      ipre[i] = acc;
      acc = JsonCompose()(acc, isum[i]);
    }
  }
  A.emit = 0;
  emu_launch(k_json_struct, grid(cap_items), block, A);
  exclusive_rows(ecnt, eoff, cap_items, 2, tot);
  if (tot[0] > cap_ev || tot[1] > cap_ev) return -100; /* the bound is broken */
  A.emit = 1;
  emu_launch(k_json_struct, grid(cap_items), block, A);
  emu_launch(k_json_packet, grid(n), block, A);
  {
    uint64_t s = 0;
    for (uint32_t k = 0; k < n; k++) {
      poff[n + k] = (uint32_t)s;
      s += pcnt[n + k];
    }
    if (s > cap_mem) return -101;
  }
  A.emit = 0;
  emu_launch(k_json_member, grid(cap_mem), block, x->S, x->W, A);
  emu_launch(k_json_fix, grid(std::max(n, cap_mem)), block, A);
  exclusive_rows(mcnt, moff, cap_mem, 3, tot);
  const uint64_t items = poff[n - 1] + pcnt[n - 1];
  if (items > cap_items) return GPX_EINVAL;
  bool small = false;
  for (int j = 0; j < 3; j++) {
    small = small || tot[j] > sizes[j];
    sizes[j] = tot[j];
  }
  if (small) return GPX_ERANGE;
  const uint32_t nr = (uint32_t)tot[1], nd = (uint32_t)tot[2];
  std::vector<gpx_accept_reply_rec> sr(nr + 1);
  std::vector<gpx_decision_rec> sd(nd + 1);
  std::vector<uint32_t> kr(nr), kd(nd);
  /* pass 1 runs without the event lists, as on the device */
  A.ev_open = A.ev_close = nullptr;
  A.mem_out = members;
  A.rep = sr.data();
  A.dec = sd.data();
  A.rep_key = kr.data();
  A.dec_key = kd.data();
  A.emit = 1;
  const uint32_t nm_all = poff[2 * n - 1] + pcnt[2 * n - 1];
  emu_launch(k_json_member, grid(nm_all), block, x->S, x->W, A);
  gather(stable_order(kr), sr, rep);
  gather(stable_order(kd), sd, dec);
  return 0;
}
