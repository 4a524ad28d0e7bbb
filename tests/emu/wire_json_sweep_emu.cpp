/*
 * wire_json_sweep_emu.cpp -- the sweep (emu_wire_encode_json_sweep) and its no-forwards form (emu_wire_encode_json),
 * both defined with the JSON-out calls in wire_json_out_emu.cpp.  Test infrastructure only.
 */
#include "wire_json_out_emu.cpp"
