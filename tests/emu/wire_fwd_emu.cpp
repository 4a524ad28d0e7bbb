/*
 * wire_fwd_emu.cpp -- gpx_wire_encode_forwards_device's and gpx_wire_decode_json_requests_device's sequences over
 * k_wire_fwd and k_json_req (gigapaxos_b200/csrc/gpx_wire_fwd.cuh) on the CPU executor, beside the byte and JSON
 * decoders of wire_json_emu.cpp (same world).  The acceptor and coordinator rows the routing reads, and the batching
 * settings, are set from the test (emu_fwd_state).  Test infrastructure only.
 */
#include "wire_json_emu.cpp"

/* sizes[2] = {bytes, refs} in / out */
extern "C" int emu_wire_encode_forwards(void* p, const gpx_request_rec* reqs, const gpx_wire_req_meta* meta, uint32_t n,
                                        const int32_t* status, const uint8_t* payload, uint32_t n_down,
                                        const int32_t* down, uint8_t* rstatus, uint8_t* out, gpx_wire_ref* refs,
                                        uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t nr = cap32(sizes[1]);
  const int rc = wire_encode_forwards(ex, call, ex.env(x->S, x->W), reqs, meta, n, status, payload, n_down, down,
                                      rstatus, out, &sizes[0], refs, &nr);
  sizes[1] = nr;
  return rc;
}

/* sizes[2] = {requests, payload bytes} in / out */
extern "C" int emu_wire_decode_json_requests(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                             const gpx_wire_ref* pkts, uint32_t n_pkts, const gpx_wire_member* mem,
                                             int64_t now_ms, int32_t* status, gpx_request_rec* reqs,
                                             gpx_wire_req_meta* meta, uint8_t* payload, uint64_t* sizes,
                                             uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t nq = cap32(sizes[0]);
  const int rc = wire_decode_json_requests(ex, call, ex.env(x->S, x->W), n, bytes, n_bytes, pkts, n_pkts, mem, now_ms,
                                           status, reqs, meta, &nq, payload, &sizes[1]);
  sizes[0] = nq;
  return rc;
}
