/*
 * wire_json_out_emu.cpp -- gpx_wire_encode_json_sweep_device's sequence over the kernels of
 * gigapaxos_b200/csrc/gpx_wire_json_enc.cuh on the CPU executor, beside the byte codec (wire_emu.cpp) and the JSON
 * decoder (wire_json_emu.cpp) on the same world.  emu_wire_encode_json is the sweep without requests, as
 * gpx_wire_encode_json_device is.  Test infrastructure only.
 */
#include "wire_json_emu.cpp"

/* sizes[2] = {bytes, refs} capacities in, sizes out.  Returns 0, GPX_ERANGE (sizes reported, no packet written) or
 * GPX_EINVAL (wrap_bytes out of range, n_replies not a multiple of n_lanes, an oversized reply or commit member). */
extern "C" int emu_wire_encode_json_sweep(void* p, uint32_t nr, const gpx_accept_reply_rec* rep,
                                          const gpx_decision_rec* dec, const uint32_t* n_dec_ptr, uint32_t nd,
                                          const gpx_request_rec* reqs, const gpx_wire_req_meta* meta, uint32_t nq,
                                          const int32_t* status, const uint8_t* payload, uint32_t n_down,
                                          const int32_t* down, uint8_t* rst_r, uint8_t* rst_d, uint8_t* rst_q,
                                          uint64_t wrap_bytes, uint8_t* out, gpx_wire_ref* refs, uint64_t* sizes,
                                          uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  JsonSetTable T; /* the recipient sets of the world's member sets, as gpx_wire_host.inc's json_sets builds them */
  T.grow(x->msets.data(), x->msets.size());
  const JsonSets Z = {T.of_mset.data(), T.one.data(), T.nodes.data(), T.count.data(), (uint32_t)T.count.size()};
  uint32_t n_refs = cap32(sizes[1]);
  const int rc = wire_encode_json_sweep(ex, call, ex.env(x->S, x->W), Z, nr, rep, dec, n_dec_ptr, nd, reqs, meta, nq,
                                        status, payload, n_down, down, rst_r, rst_d, rst_q, wrap_bytes, out, &sizes[0],
                                        refs, &n_refs);
  sizes[1] = n_refs;
  return rc;
}

extern "C" int emu_wire_encode_json(void* p, uint32_t nr, const gpx_accept_reply_rec* rep, const gpx_decision_rec* dec,
                                    const uint32_t* n_dec_ptr, uint32_t nd, uint8_t* rst_r, uint8_t* rst_d,
                                    uint64_t wrap_bytes, uint8_t* out, gpx_wire_ref* refs, uint64_t* sizes,
                                    uint32_t block) {
  return emu_wire_encode_json_sweep(p, nr, rep, dec, n_dec_ptr, nd, nullptr, nullptr, 0, nullptr, nullptr, 0, nullptr,
                                    rst_r, rst_d, nullptr, wrap_bytes, out, refs, sizes, block);
}
