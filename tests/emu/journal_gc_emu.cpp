/*
 * journal_gc_emu.cpp -- the journal GC kernels (gigapaxos_b200/csrc/gpx_journal_gc.cuh, the source the GPU runs)
 * compiled for the host over cuda_emu.h, and driven by the product's own host sequence (journal_compact in
 * gpx_wire_seq.h) on the CPU executor of wire_exec.h.  The caller hands in the name table's contents and which groups
 * are live; gpx_journal_index's walk is the same function the engine exports.  Test infrastructure only.
 */
#include "wire_exec.h"

struct EmuJournalGc {
  DevState S;
  WireNames W;
  std::vector<uint2> tab;
  std::vector<uint8_t> name;
  std::vector<int32_t> version;
  std::vector<uint32_t> slot, meta;
  std::vector<MsetInfo> msets;
};

/* an engine of G groups, none live and none named */
extern "C" void* emu_jgc_new(uint32_t G) {
  EmuJournalGc* x = new EmuJournalGc();
  memset(&x->S, 0, sizeof x->S);
  x->S.G = G;
  x->S.L = 1;
  x->meta.assign(G, 0);
  x->msets.resize(1);
  memset(x->msets.data(), 0, sizeof(MsetInfo));
  x->S.grp_meta = x->meta.data();
  x->S.msets = x->msets.data();
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
extern "C" void emu_jgc_free(void* p) { delete static_cast<EmuJournalGc*>(p); }

/* names staged as [n][GPX_NAME_BYTES] (length byte + bytes), version[k] for gids[k], as gpx_set_group_names stores
 * them; live[k] sets the group's liveness */
extern "C" void emu_jgc_names(void* p, uint32_t n, const uint32_t* gids, const uint8_t* staged, const int32_t* version,
                              const uint8_t* live) {
  EmuJournalGc* x = static_cast<EmuJournalGc*>(p);
  NameSetArgs A;
  A.gids = gids;
  A.n = n;
  emu_launch(k_names_remove, (n + 63) / 64, 64, x->W, A);
  emu_launch(k_names_store, (n + 63) / 64, 64, x->W, A, staged, version);
  emu_launch(k_names_insert, (n + 63) / 64, 64, x->W, A);
  for (uint32_t k = 0; k < n; k++) x->meta[gids[k]] = live[k] ? GPX_META_LIVE : 0u;
}

/* gpx_journal_compact_device: sizes[2] = {out bytes, bad} are capacities in, sizes out */
extern "C" int emu_jgc_compact(void* p, const uint8_t* bytes, uint64_t n_bytes, const uint32_t* file_off,
                               uint32_t n_files, const uint32_t* starts, uint32_t n, const int32_t* gc_slot,
                               uint32_t n_gids, uint32_t last_readonly, uint8_t* out, gpx_journal_file* files,
                               uint32_t* bad, uint64_t* sizes, uint32_t block) {
  EmuJournalGc* x = static_cast<EmuJournalGc*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t nb = cap32(sizes[1]);
  const int rc = journal_compact(ex, call, ex.env(x->S, x->W), bytes, n_bytes, file_off, n_files, starts, n, gc_slot,
                                 n_gids, last_readonly, out, &sizes[0], files, bad, &nb);
  sizes[1] = nb;
  return rc;
}

extern "C" int emu_jgc_index(const uint8_t* buf, uint64_t n_bytes, uint32_t base, uint32_t* starts, uint32_t cap,
                             uint32_t* n_frames, uint64_t* end) {
  return journal_index(buf, n_bytes, base, starts, cap, n_frames, end);
}
