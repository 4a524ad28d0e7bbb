/*
 * journal_emu.cpp -- the journal frame kernels (gigapaxos_b200/csrc/gpx_journal.cuh and the k_log_dir walk they reuse,
 * the source the GPU runs) compiled for the host over cuda_emu.h, and driven by the product's own host sequence
 * (log_frame in gpx_wire_seq.h) on the CPU executor of wire_exec.h.  The caller hands in one lane's ring as the device
 * holds it (ring_cap bytes, positions taken modulo ring_cap), the head and the name table's contents.  Test
 * infrastructure only.
 */
#include "wire_exec.h"

struct EmuJournal {
  DevState S;
  WireNames W;
  std::vector<uint2> tab;
  std::vector<uint8_t> name;
  std::vector<int32_t> version;
  std::vector<uint32_t> slot;
  std::vector<unsigned long long> ctr, log_pos;
};

/* an engine of G groups whose lane `lane` logs; no gid has a name until emu_journal_names */
extern "C" void* emu_journal_new(uint32_t G, uint32_t lane) {
  if (lane >= GPX_MAX_LANES) return nullptr;
  EmuJournal* x = new EmuJournal();
  memset(&x->S, 0, sizeof x->S);
  x->S.G = G;
  x->S.L = lane + 1;
  x->ctr.assign((size_t)GPX_CTR_STRIPES * C_NCTR, 0ull);
  x->log_pos.assign((size_t)2 * GPX_MAX_LANES * 2, 0ull);
  x->S.ctr = x->ctr.data();
  x->S.log_pos = x->log_pos.data();
  x->S.lp = 1; /* the copy the next launch would read */
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
extern "C" void emu_journal_free(void* p) { delete static_cast<EmuJournal*>(p); }

/* names staged as [n][GPX_NAME_BYTES] (length byte + bytes), version[k] for gids[k], as gpx_set_group_names stores
 * them; n = 0 with gids removes nothing */
extern "C" void emu_journal_names(void* p, uint32_t n, const uint32_t* gids, const uint8_t* staged,
                                  const int32_t* version) {
  EmuJournal* x = static_cast<EmuJournal*>(p);
  NameSetArgs A;
  A.gids = gids;
  A.n = n;
  emu_launch(k_names_remove, (n + 63) / 64, 64, x->W, A);
  emu_launch(k_names_store, (n + 63) / 64, 64, x->W, A, staged, version);
  emu_launch(k_names_insert, (n + 63) / 64, 64, x->W, A);
}
extern "C" void emu_journal_names_remove(void* p, uint32_t n, const uint32_t* gids) {
  EmuJournal* x = static_cast<EmuJournal*>(p);
  NameSetArgs A;
  A.gids = gids;
  A.n = n;
  emu_launch(k_names_remove, (n + 63) / 64, 64, x->W, A);
}

/* gpx_log_frame_device on the ring image: sizes[3] = {frame bytes, frames, misses} are capacities in, sizes out */
extern "C" int emu_log_frame(void* p, uint8_t* ring, uint64_t ring_cap, uint64_t head, uint64_t* from,
                             const gpx_journal_req* meta, uint32_t n_meta, uint8_t* out, gpx_journal_miss* missing,
                             uint64_t* sizes, uint32_t block) {
  EmuJournal* x = static_cast<EmuJournal*>(p);
  if (ring_cap & (ring_cap - 1)) return -100;
  const uint32_t lane = x->S.L - 1;
  x->S.ring[lane] = ring;
  x->S.ring_cap = ring_cap;
  x->log_pos[((size_t)x->S.lp * GPX_MAX_LANES + lane) * 2] = head;
  EmuExec ex{block};
  EmuCall call;
  uint32_t nf = cap32(sizes[1]), nm = cap32(sizes[2]);
  const int rc = log_frame(ex, call, ex.env(x->S, x->W), lane, from, head, meta, n_meta, out, &sizes[0], &nf, missing,
                           &nm);
  sizes[1] = nf;
  sizes[2] = nm;
  return rc;
}
