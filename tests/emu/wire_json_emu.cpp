/*
 * wire_json_emu.cpp -- gpx_wire_decode_json_device's sequence over the JSON decoder's kernels
 * (gigapaxos_b200/csrc/gpx_wire_json.cuh) on the CPU executor, beside the byte codec of wire_emu.cpp (same world).
 * Build with -DGPX_JSON_CHUNK=<bytes> to cut packets into chunks that small.  Test infrastructure only.
 */
#include "wire_emu.cpp"

/* sizes[3] = {members, replies, decisions} capacities in, sizes out.  Returns 0, GPX_ERANGE (an output too small),
 * GPX_EINVAL (the lengths exceed the arena) or EMU_EBOUND (more events or members than the host's bounds) */
extern "C" int emu_wire_decode_json(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                    const gpx_wire_ref* pkts, int32_t* status, gpx_wire_member* members,
                                    gpx_accept_reply_rec* rep, gpx_decision_rec* dec, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t nm = cap32(sizes[0]), nr = cap32(sizes[1]), nd = cap32(sizes[2]);
  const int rc = wire_decode_json(ex, call, ex.env(x->S, x->W), n, bytes, n_bytes, pkts, status, members, &nm, rep,
                                  &nr, dec, &nd);
  sizes[0] = nm;
  sizes[1] = nr;
  sizes[2] = nd;
  return rc;
}
