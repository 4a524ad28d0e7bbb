/*
 * wire_emu.cpp -- k_names_*, k_wire_decode, k_wire_req_decode and the k_wire_enc_* kernels
 * (gigapaxos_b200/csrc/gpx_wire_dev.cuh, the source the GPU runs) compiled for the host over cuda_emu.h; see
 * p1b_emu.cpp.  The scans and the stable sorts by gid that gpx_wire_host.inc does with CUB are done here with the
 * standard library.  Test infrastructure only.
 */
#include "cuda_emu.h"

template <class T>
static inline T atomicCAS(T* p, T cmp, T v) { /* one thread at a time */
  T old = *p;
  if (old == cmp) *p = v;
  return old;
}

#include "gpx_wire_dev.cuh"

#include <numeric>
#include <vector>

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

static std::vector<uint32_t> stable_order(const std::vector<uint32_t>& key) {
  std::vector<uint32_t> perm(key.size());
  std::iota(perm.begin(), perm.end(), 0u);
  std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) { return key[a] < key[b]; });
  return perm;
}
/* records into a stable order: dst[i] = src[perm[i]] */
template <class T>
static void gather(const std::vector<uint32_t>& perm, const std::vector<T>& src, T* dst) {
  for (size_t i = 0; i < perm.size(); i++) dst[i] = src[perm[i]];
}
static void exclusive_rows(const std::vector<uint32_t>& cnt, std::vector<uint32_t>& off, uint32_t n, uint32_t rows,
                           uint64_t* tot) {
  for (uint32_t j = 0; j < rows; j++) {
    uint64_t s = 0;
    for (uint32_t i = 0; i < n; i++) {
      off[(size_t)j * n + i] = (uint32_t)s;
      s += cnt[(size_t)j * n + i];
    }
    tot[j] = s;
  }
}

/* gpx_wire_decode_batch without the copies; sizes[4] = {accepts, blob bytes, replies, decisions} are capacities in,
 * sizes out; returns -5 (GPX_ERANGE) when an output is too small */
extern "C" int emu_wire_decode(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes, const gpx_wire_ref* pkts,
                               int32_t* status, gpx_accept_rec* acc, uint8_t* blob, gpx_accept_reply_rec* rep,
                               gpx_decision_rec* dec, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  std::vector<uint32_t> cnt((size_t)WD_NCNT * n + 1), off((size_t)WD_NCNT * n + 1);
  WireDecodeArgs A;
  memset(&A, 0, sizeof A);
  A.bytes = bytes;
  A.pkts = pkts;
  A.n_bytes = n_bytes;
  A.n = n;
  A.cnt = cnt.data();
  A.off = off.data();
  A.status = status;
  emu_launch(k_wire_decode, (n + block - 1) / block, block, x->S, x->W, A);
  uint64_t tot[WD_NCNT];
  exclusive_rows(cnt, off, n, WD_NCNT, tot);
  bool small = false;
  for (int j = 0; j < WD_NCNT; j++) {
    small = small || tot[j] > sizes[j];
    sizes[j] = tot[j];
  }
  if (small) return GPX_ERANGE;
  std::vector<gpx_accept_rec> sa(tot[WD_ACC] + 1);
  std::vector<gpx_accept_reply_rec> sr(tot[WD_REP] + 1);
  std::vector<gpx_decision_rec> sd(tot[WD_DEC] + 1);
  std::vector<uint32_t> ka(tot[WD_ACC]), kr(tot[WD_REP]), kd(tot[WD_DEC]);
  A.acc = sa.data();
  A.blob = blob;
  A.rep = sr.data();
  A.dec = sd.data();
  A.acc_key = ka.data();
  A.rep_key = kr.data();
  A.dec_key = kd.data();
  A.emit = 1;
  emu_launch(k_wire_decode, (n + block - 1) / block, block, x->S, x->W, A);
  gather(stable_order(ka), sa, acc);
  gather(stable_order(kr), sr, rep);
  gather(stable_order(kd), sd, dec);
  return 0;
}

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
  const std::vector<uint32_t> perm = stable_order(key);
  gather(perm, sq, reqs);
  gather(perm, sm, meta);
  return 0;
}

enum { EMU_ENC_REPLIES = 0, EMU_ENC_DECISIONS = 1, EMU_ENC_ACCEPTS = 2 };

/* gpx_wire_encode_replies (kind 0: n records of n_lanes), gpx_wire_encode_decisions (1) or
 * gpx_wire_encode_accepts_device (2, the ACCEPTs' requests at heads .. payload) without the copies.  The keys, the sort
 * and the passes run over n records; n_ptr, when not null, is the record count as the device reads it.  sizes[2] =
 * {bytes, refs} in / out. */
extern "C" int emu_wire_encode(void* p, int kind, const uint32_t* n_ptr, uint32_t n, const void* recs,
                               const uint32_t* heads, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta,
                               uint32_t n_reqs, const uint8_t* payload, uint8_t* rstatus, uint8_t* out,
                               gpx_wire_ref* refs, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
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
  const uint32_t grid = (n + block - 1) / block;
  const auto launch = [&](bool keys) {
    if (kind == EMU_ENC_REPLIES)
      keys ? emu_launch(k_wire_enc_keys_replies, grid, block, x->S, x->W, A)
           : emu_launch(k_wire_enc_replies, grid, block, x->S, x->W, A);
    else if (kind == EMU_ENC_DECISIONS)
      keys ? emu_launch(k_wire_enc_keys_decisions, grid, block, x->S, x->W, A)
           : emu_launch(k_wire_enc_decisions, grid, block, x->S, x->W, A);
    else
      keys ? emu_launch(k_wire_enc_keys_accepts, grid, block, x->S, x->W, A, X)
           : emu_launch(k_wire_enc_accepts, grid, block, x->S, x->W, A, X);
  };
  launch(true);
  key.resize(n);
  perm = stable_order(key);
  for (uint32_t i = 0; i < n; i++) skey[i] = key[perm[i]];
  A.perm = perm.data();
  A.skey = skey.data();
  A.cnt = cnt.data();
  A.off = off.data();
  launch(false);
  uint64_t tot[2];
  exclusive_rows(cnt, off, n, 2, tot);
  const bool small = tot[0] > sizes[0] || tot[1] > sizes[1];
  sizes[0] = tot[0];
  sizes[1] = tot[1];
  if (small) return GPX_ERANGE;
  A.out = out;
  A.refs = refs;
  A.emit = 1;
  launch(false);
  return 0;
}
