/*
 * wire_emu.cpp -- the wire calls' kernels (gigapaxos_b200/csrc/gpx_wire_*.cuh, the source the GPU runs) compiled for the
 * host over cuda_emu.h, and driven by the product's own host sequences (gpx_wire_seq.h) on the CPU executor of
 * wire_exec.h.  This file holds the world the kernels read (engine state, member sets, the name table) and the byte
 * codec's calls; wire_json_emu.cpp, wire_fwd_emu.cpp, wire_json_out_emu.cpp and wire_json_sweep_emu.cpp add the
 * others over the same world.  Test infrastructure only.
 */
#include "wire_exec.h"

struct EmuWire {
  DevState S;
  WireNames W;
  std::vector<MsetInfo> msets;
  std::vector<uint32_t> meta;
  std::vector<uint2> tab;
  std::vector<uint8_t> name;
  std::vector<int32_t> version;
  std::vector<uint32_t> slot;
};

/* an engine of G groups and L lanes serving lane_node[]; no group is live until emu_wire_group */
extern "C" void* emu_wire_new(uint32_t G, uint32_t L, const int32_t* lane_node) {
  EmuWire* x = new EmuWire();
  memset(&x->S, 0, sizeof x->S);
  x->S.G = G;
  x->S.L = L;
  for (uint32_t l = 0; l < GPX_MAX_LANES; l++) x->S.lane_node[l] = l < L ? lane_node[l] : INT32_MIN;
  x->meta.assign(G, 0);
  x->msets.reserve(GPX_MAX_MSETS);
  MsetInfo none; /* member set 0: what the grp_meta of a group that is not live points at */
  memset(&none, 0xff, sizeof none);
  none.R = 0;
  none.lane_mask = 0;
  x->msets.push_back(none);
  x->S.msets = x->msets.data();
  x->S.grp_meta = x->meta.data();
  size_t cap = 1024;
  while (cap < 2 * (size_t)G) cap <<= 1;
  x->tab.assign(cap, make_uint2(0, 0));
  x->name.assign((size_t)G * GPX_NAME_BYTES, 0);
  x->version.assign(G, 0);
  x->slot.assign(G, GPX_NAME_NONE);
  x->W.tab = x->tab.data();
  x->W.mask = (uint32_t)(cap - 1);
  x->W.name = x->name.data();
  x->W.version = x->version.data();
  x->W.slot = x->slot.data();
  return x;
}
extern "C" void emu_wire_free(void* p) { delete static_cast<EmuWire*>(p); }

/* live group gid with members m[0..R) (sorted ascending), as gpx_create_groups' intern_mset lays it out */
extern "C" int emu_wire_group(void* p, uint32_t gid, uint32_t R, const int32_t* m) {
  EmuWire* x = static_cast<EmuWire*>(p);
  if (gid >= x->S.G || R == 0 || R > GPX_MAX_GROUP_SIZE || x->msets.size() >= GPX_MAX_MSETS) return -1;
  MsetInfo mi;
  memset(&mi, 0xff, sizeof mi);
  mi.R = (uint8_t)R;
  mi.lane_mask = 0;
  mi.ident = 0;
  mi.pad2 = 0;
  for (uint32_t i = 0; i < GPX_MAX_GROUP_SIZE; i++) mi.nodes[i] = i < R ? m[i] : INT32_MIN;
  for (uint32_t l = 0; l < x->S.L; l++)
    for (uint32_t i = 0; i < R; i++)
      if (m[i] == x->S.lane_node[l]) {
        mi.lane_of_idx[i] = (uint8_t)l;
        mi.idx_of_lane[l] = (uint8_t)i;
        mi.lane_mask |= (uint16_t)(1u << l);
      }
  x->msets.push_back(mi);
  x->meta[gid] = (uint32_t)(x->msets.size() - 1) | (R << 16) | GPX_META_LIVE;
  x->S.msets = x->msets.data();
  x->S.grp_meta = x->meta.data();
  return 0;
}

/* names staged as [n][GPX_NAME_BYTES]; version[k] for gids[k]: remove, store, insert (as gpx_set_group_names) */
extern "C" void emu_wire_names(void* p, uint32_t n, const uint32_t* gids, const uint8_t* staged, const int32_t* version,
                               uint32_t* found) {
  EmuWire* x = static_cast<EmuWire*>(p);
  NameSetArgs A;
  A.gids = gids;
  A.n = n;
  emu_launch(k_names_find, (n + 63) / 64, 64, x->W, staged, n, found);
  emu_launch(k_names_remove, (n + 63) / 64, 64, x->W, A);
  emu_launch(k_names_store, (n + 63) / 64, 64, x->W, A, staged, version);
  emu_launch(k_names_insert, (n + 63) / 64, 64, x->W, A);
}
extern "C" void emu_wire_names_remove(void* p, uint32_t n, const uint32_t* gids) {
  EmuWire* x = static_cast<EmuWire*>(p);
  NameSetArgs A;
  A.gids = gids;
  A.n = n;
  emu_launch(k_names_remove, (n + 63) / 64, 64, x->W, A);
}
extern "C" void emu_wire_names_rehash(void* p) {
  EmuWire* x = static_cast<EmuWire*>(p);
  std::fill(x->tab.begin(), x->tab.end(), make_uint2(0, 0));
  emu_launch(k_names_rehash, (x->S.G + 63) / 64, 64, x->W, x->S.G);
}

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

/* gpx_wire_decode_batch_device; sizes[4] = {accepts, blob bytes, replies, decisions} are capacities in, sizes out */
extern "C" int emu_wire_decode(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes, const gpx_wire_ref* pkts,
                               int32_t* status, gpx_accept_rec* acc, uint8_t* blob, gpx_accept_reply_rec* rep,
                               gpx_decision_rec* dec, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t na = cap32(sizes[0]), nr = cap32(sizes[2]), nd = cap32(sizes[3]);
  const int rc = wire_decode(ex, call, ex.env(x->S, x->W), n, bytes, n_bytes, pkts, status, acc, &na, blob, &sizes[1],
                             rep, &nr, dec, &nd);
  sizes[0] = na;
  sizes[2] = nr;
  sizes[3] = nd;
  return rc;
}

/* gpx_wire_decode_requests_device; sizes[2] = {requests, payload bytes} in / out */
extern "C" int emu_wire_decode_requests(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                        const gpx_wire_ref* pkts, int64_t now_ms, int32_t* status,
                                        gpx_request_rec* reqs, gpx_wire_req_meta* meta, uint8_t* payload,
                                        uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t nq = cap32(sizes[0]);
  const int rc = wire_decode_requests(ex, call, ex.env(x->S, x->W), n, bytes, n_bytes, pkts, now_ms, status, reqs, meta,
                                      &nq, payload, &sizes[1]);
  sizes[0] = nq;
  return rc;
}

/* gpx_wire_encode_replies_device (kind 0: n records of n_lanes), gpx_wire_encode_decisions_device (1) or
 * gpx_wire_encode_accepts_device (2, the ACCEPTs' requests at heads .. payload); n_ptr, when not null, is the record
 * count as the device reads it.  sizes[2] = {bytes, refs} in / out. */
extern "C" int emu_wire_encode(void* p, int kind, const uint32_t* n_ptr, uint32_t n, const void* recs,
                               const uint32_t* heads, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta,
                               uint32_t n_reqs, const uint8_t* payload, uint8_t* rstatus, uint8_t* out,
                               gpx_wire_ref* refs, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  /* with a device count of 0 a test may hand in no records and no heads at all; the entry point wants buffers there,
   * so empty ones stand in, and AddressSanitizer traps any read of them */
  const std::unique_ptr<uint32_t[]> none(new uint32_t[0]);
  if (!recs) recs = none.get();
  if (!heads) heads = none.get();
  WireAccArgs Q;
  Q.head = heads;
  Q.reqs = reqs;
  Q.meta = meta;
  Q.n_reqs = n_reqs;
  Q.payload = payload;
  uint32_t nr = cap32(sizes[1]);
  const int rc = wire_encode(ex, call, ex.env(x->S, x->W), (WireEnc)kind, n, n_ptr, recs, Q, rstatus, out, &sizes[0],
                             refs, &nr);
  sizes[1] = nr;
  return rc;
}
