/*
 * wire_client_emu.cpp -- gpx_wire_decode_client_requests_device's sequence over k_json_client
 * (gigapaxos_b200/csrc/gpx_wire_fwd.cuh) on the CPU executor, beside the byte, JSON and JSON-request decoders of
 * wire_fwd_emu.cpp (same world).  Test infrastructure only.
 */
#include "wire_fwd_emu.cpp"

/* sizes[2] = {requests, payload bytes} in / out; peers may be null */
extern "C" int emu_wire_decode_client_requests(void* p, uint32_t n, const uint8_t* bytes, uint64_t n_bytes,
                                               const gpx_wire_ref* pkts, const gpx_wire_peer* peers, int64_t now_ms,
                                               int32_t* status, gpx_request_rec* reqs, gpx_wire_req_meta* meta,
                                               uint8_t* payload, uint64_t* sizes, uint32_t block) {
  EmuWire* x = static_cast<EmuWire*>(p);
  EmuExec ex{block};
  EmuCall call;
  uint32_t nq = cap32(sizes[0]);
  const int rc = wire_decode_client_requests(ex, call, ex.env(x->S, x->W), n, bytes, n_bytes, pkts, peers, now_ms,
                                             status, reqs, meta, &nq, payload, &sizes[1]);
  sizes[0] = nq;
  return rc;
}
