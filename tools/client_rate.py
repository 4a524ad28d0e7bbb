#!/usr/bin/env python3
"""Rate of gpx_wire_decode_client_requests_device: a node's front door for a Java client's own REQUEST packets.

For n client packets of bench.py cfg2's shape (one 1-byte request per group, n groups, org.json with no "CA", each
packet's connection in a gpx_wire_peer row), in one run:

* client       gpx_wire_decode_client_requests_device on the device-resident arena, refs and peers;
* client+up    the same with the upload of the arena, refs and peers from pinned host memory before it;
* json_req     gpx_wire_decode_json_requests_device over the same requests with "CA" / "LA" written out, as whole-packet
               members (what the call did before a client's packet had a device form, given a host that inserted the
               addresses);
* host         json.loads of every packet and its fields into request records, with the connection's address: the host
               path the call replaces (one Python loop; its records are compared with the device's).

Wall figures are the best of --reps runs to a device synchronise, after a warm-up run of the same shape; the legs
alternate.  Kernel time is the sum of the CUDA kernels torch.profiler records over one more call, in a separate profiled
run.  The outputs of client and json_req are compared byte for byte.  The card's name, power limit and SM clock are read
in the same run (nvidia-smi --query-gpu, read only).

    python tools/client_rate.py [--packets 100000 1000000] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from wire_rate import card_info, kernel_ms  # noqa: E402

NOW = 1_700_000_000_000


def host_decode(pkts, peers, by_name):
    """json.loads per packet into (gid, req_id, entry_time, client ip/port) rows: the host's work per client packet"""
    out = np.zeros(len(pkts), [("gid", "<u4"), ("req_id", "<i8"), ("entry_time", "<i8"), ("client_port", "<u2")])
    for k, b in enumerate(pkts):
        d = json.loads(b.decode("iso-8859-1"))
        out[k] = (by_name[d["ID"]], d["QID"], NOW if d["E"] == -1 else d["ET"],
                  int(peers[k]["sender_port"]) if "CA" not in d else 0)
    return out


def run(lib, n, reps, profile):
    import torch

    from gigapaxos_b200 import abi, wire
    from helpers import Engine, group_descs_fast, make_config
    from wire_client_cases import bulk_client_packets
    G = n
    e = Engine(lib, make_config(lib, max_groups=G, n_lanes=3, lane_node=[100, 101, 102], max_batch_recs=G,
                                max_batch_payload=16 * G, log_ring_bytes=1 << 20))
    e.create_groups(group_descs_fast(G))
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    wire.set_group_names(e, np.arange(G), names)
    plain, inserted, peers = bulk_client_packets(n, G, np.random.default_rng(n))

    def packed(pkts):
        arena, refs = wire.pack_packets(pkts)
        refs["node"] = 100
        return arena, refs
    arena, refs = packed(plain)
    ia, ir = packed(inserted)
    mem = np.zeros(n, abi.wire_member_dtype)
    mem["pkt"], mem["off"], mem["len"], mem["status"] = np.arange(n), ir["off"], ir["len"], abi.WS_UNHANDLED
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).to("cuda")
    h_arena, h_refs, h_peers = (torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).pin_memory()
                                for a in (arena, refs, peers))
    d_arena, d_refs, d_peers = dev(arena), dev(refs).view(n, 16), dev(peers).view(n, 16)
    d_ia, d_ir, d_mem = dev(ia), dev(ir).view(n, 16), dev(mem).view(n, 16)
    caps = (n, 16 * n)

    legs = {
        "client": lambda: wire.decode_client_requests_device(e, d_arena, d_refs, d_peers, NOW, caps),
        "client+up": lambda: wire.decode_client_requests_device(
            e, h_arena.to("cuda", non_blocking=True), h_refs.to("cuda", non_blocking=True).view(n, 16),
            h_peers.to("cuda", non_blocking=True).view(n, 16), NOW, caps),
        "json_req": lambda: wire.decode_json_requests_device(e, d_ia, d_ir, d_mem, n, NOW, caps),
    }
    walls = {k: [] for k in legs}
    outs = {}
    for r in range(reps + 1):
        for k, fn in legs.items():
            torch.cuda.synchronize()
            t = time.perf_counter()
            outs[k] = fn()
            torch.cuda.synchronize()
            if r:
                walls[k].append(time.perf_counter() - t)
    a, b = outs["client"], outs["json_req"]
    same = (a.sizes == b.sizes and bool((a.status == abi.WS_OK).all()) and torch.equal(a.status, b.status)
            and torch.equal(a.reqs, b.reqs) and torch.equal(a.meta, b.meta) and torch.equal(a.payload, b.payload))
    by_name = {s: g for g, s in enumerate(names)}
    t = time.perf_counter()
    host = host_decode(plain, peers, by_name)
    host_s = time.perf_counter() - t
    got = wire.to_records(a.reqs, abi.request_dtype)
    same_host = np.array_equal(np.sort(host["req_id"]), np.sort(got["req_id"]))
    res = {"packets": n, "arena_bytes": int(len(arena)), "outputs_equal_json_req": same, "host_records_equal": same_host}
    for k, w in walls.items():
        res[f"{k}_ms"] = round(min(w) * 1e3, 3)
        res[f"{k}_Mpkt_s"] = round(n / min(w) / 1e6, 2)
    res["host_ms"] = round(host_s * 1e3, 1)
    res["host_Mpkt_s"] = round(n / host_s / 1e6, 3)
    if profile:
        res["client_kernel_ms"] = round(kernel_ms(legs["client"]), 3)
        res["json_req_kernel_ms"] = round(kernel_ms(legs["json_req"]), 3)
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--packets", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import gigapaxos_b200
    lib = gigapaxos_b200.load_library()
    out = {"card": card_info(), "results": [run(lib, n, args.reps, not args.no_profile) for n in args.packets]}
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
