#!/usr/bin/env python3
"""Rates of the forwarding wire calls, on the two chains a forwarded client request takes.

* forward_chain -- a non-coordinator (node 101 of groups {100, 101, 102}) with one client REQUEST per group that
  another node coordinates.  Device leg: one upload of the request arena, gpx_wire_decode_requests_device ->
  gpx_propose_device_heads -> gpx_wire_encode_forwards_device, one download of the forwarded packets.  Host leg: the
  same requests through gpx_propose (host records) and the per-packet host codec (wire.encode_request, one call per
  forward), on a second engine in the same state.  Both must write the same packets.
* json_chain -- a coordinator (node 100) receiving a Java peer's forwards: one JSON REQUEST member per group it
  coordinates, in 4 MiB BATCHED_PAXOS_PACKET wrappers.  Device leg: one upload, gpx_wire_decode_json_device ->
  gpx_wire_decode_json_requests_device -> gpx_propose_device_heads -> gpx_wire_encode_accepts_device, one download
  of the ACCEPT packets.  Host leg: json.loads of the wrappers, the members into request records, gpx_propose and the
  per-packet host encoder (wire.encode_accept).  Both must write the same ACCEPT packets.

The legs alternate in one run; each figure is the best of --reps wall times to a device synchronise (a warm-up round
first).  Kernel time is the sum of the CUDA kernels torch.profiler records over one more device round, in a separate
profiled run.  The card's name, power limit and SM clock are read in the same run (nvidia-smi --query-gpu, read only).

    python tools/forward_rate.py [--groups 100000 1000000] [--reps 5] [--out FILE]
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

MEMBERS = [100, 101, 102]
NOW = 1_700_000_000_000
WRAP_BYTES = 4 << 20  # a Java peer's wrapper is at most 4 MiB


def engines(lib, G, node, gids, names, n=2):
    from gigapaxos_b200 import wire
    from helpers import Engine, group_descs_fast, make_config
    out = []
    for _ in range(n):
        e = Engine(lib, make_config(lib, max_groups=G, n_lanes=1, lane_node=[node], window=8, max_batch_recs=G,
                                    max_batch_payload=16 * G, log_ring_bytes=1 << 20))
        e.create_groups(group_descs_fast(G, members=tuple(MEMBERS)))
        wire.set_group_names(e, gids, [names[g] for g in gids])
        out.append(e)
    return out


def alternate(legs, rounds, check):
    """run the legs alternately over rounds 0..rounds-1 (round 0 warms up); the best wall time of each leg"""
    walls = {k: [] for k in legs}
    for r in range(rounds):
        outs = {}
        for k, run in legs.items():
            t = time.perf_counter()
            outs[k] = run(r)
            if r:
                walls[k].append(time.perf_counter() - t)
        check(r, outs)
    return {k: min(v) for k, v in walls.items()}


def forward_chain(lib, G, reps, profile):
    import torch

    from gigapaxos_b200 import abi, wire
    from gigapaxos_b200.spread import coordinator_of

    names = [f"NoopPaxosApp{i}" for i in range(G)]
    coord = np.array([coordinator_of(s, MEMBERS) for s in names])
    gids = np.nonzero(coord != 101)[0].astype(np.uint32)
    ed, eh = engines(lib, G, 101, np.arange(G, dtype=np.uint32), names)
    n = len(gids)

    def round_requests(r):
        return [wire.Request(names[g], 0, r * G + int(g), b"12345678", client=("10.0.0.1", 2000)) for g in gids]

    rounds = []
    for r in range(reps + 2):
        reqs = round_requests(r)
        arena, refs = wire.pack_packets([wire.encode_request(q) for q in reqs])
        refs["node"] = 101
        rounds.append((torch.from_numpy(arena.copy()).pin_memory(),
                       torch.from_numpy(refs.view(np.uint8).reshape(n, 16).copy()).pin_memory(), reqs))
    d_arena = torch.empty(rounds[0][0].numel(), dtype=torch.uint8, device="cuda")
    d_refs = torch.empty((n, 16), dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    acc = torch.empty((n, 48), dtype=torch.uint8, device="cuda")
    heads = torch.empty(n, dtype=torch.int32, device="cuda")
    ctl = torch.zeros(8, dtype=torch.int32, device="cuda")
    h_out = torch.empty(128 * n, dtype=torch.uint8).pin_memory()
    h_refs = torch.empty((n, 16), dtype=torch.uint8).pin_memory()
    caps = {"req": (n, 16 * n), "fwd": (128 * n, n)}

    def device_leg(r):
        d_arena.copy_(rounds[r][0], non_blocking=True)
        d_refs.copy_(rounds[r][1], non_blocking=True)
        d = wire.decode_requests_device(ed, d_arena, d_refs, NOW, caps["req"])
        ctl.zero_()
        wire.propose_device_heads(ed, d.reqs, d.sizes[0], d.payload, d.sizes[1], status, acc, heads, ctl)
        f = wire.encode_forwards_device(ed, d.reqs, d.meta, d.sizes[0], status, d.payload, [], caps["fwd"])
        caps["req"], caps["fwd"] = d.sizes, f.sizes
        h_out[: f.sizes[0]].copy_(f.out, non_blocking=True)
        h_refs[: f.sizes[1]].copy_(f.refs, non_blocking=True)
        torch.cuda.synchronize()
        return f.sizes

    pay = np.zeros(16 * n, np.uint8)
    pay.reshape(n, 16)[:, :8] = np.frombuffer(b"12345678", np.uint8)
    host_reqs = np.zeros(n, abi.request_dtype)
    host_reqs["gid"], host_reqs["payload_off"], host_reqs["payload_len"] = gids, 16 * np.arange(n), 8
    host_reqs["entry_node"], host_reqs["client"] = 101, np.arange(n)

    def host_leg(r):
        reqs = host_reqs.copy()
        reqs["req_id"] = r * G + gids.astype(np.int64)
        _, _, st = eh.propose(reqs, pay)
        out = []
        for k in np.nonzero(st == abi.RS_FORWARD)[0]:  # a forward per request: one request per group
            q = rounds[r][2][int(k)]
            q.entry_replica, q.entry_time, q.forward_count = 101, NOW, 1
            out.append(wire.encode_request(q))
        return out

    def check(r, outs):
        refs = h_refs[: outs["device"][1]].numpy().reshape(-1).view(abi.wire_ref_dtype)
        got = [bytes(h_out[int(x["off"]): int(x["off"]) + int(x["len"])].numpy()) for x in refs]
        assert got == outs["host"] and len(got) == n, "device and host forwards differ"

    res = {"groups": G, "requests": n}
    if profile:
        device_leg(0)
        res["device_kernel_ms"] = min(kernel_ms(lambda: device_leg(r)) for r in range(1, reps + 1))
        res["requests_per_s_kernels"] = n / (res["device_kernel_ms"] / 1000.0)
    else:
        w = alternate({"device": device_leg, "host": host_leg}, reps + 1, check)
        for leg, s in w.items():
            res[leg] = {"wall_s_min": s, "requests_per_s_wall": n / s}
    res["forward_bytes"] = int(caps["fwd"][0])
    for e in (ed, eh):
        e.close()
    return res


def json_chain(lib, G, reps, profile):
    import torch

    from gigapaxos_b200 import abi, packets_json as pj, wire
    from gigapaxos_b200.spread import coordinator_of

    assert reps + 2 <= 8, "every round takes a slot of the window"
    names = [f"NoopPaxosApp{i}" for i in range(G)]
    coord = np.array([coordinator_of(s, MEMBERS) for s in names])
    gids = np.nonzero(coord == 100)[0].astype(np.uint32)
    ed, eh = engines(lib, G, 100, gids, names)
    n = len(gids)

    def round_requests(r):  # as node 101 forwards them: entered there, forwarded once
        return [wire.Request(names[g], 0, r * G + int(g), b"12345678", client=("10.0.0.1", 2000), entry_replica=101,
                             entry_time=NOW, forward_count=1) for g in gids]

    rounds = []
    for r in range(reps + 2):
        reqs = round_requests(r)
        members = [pj.request_json(q) for q in reqs]
        wraps, cur, size = [], [], 0
        for m in members:
            if cur and size + len(m) + 64 > WRAP_BYTES:
                wraps.append(b'{"type":90,"PT":37,"V":-1,"PP":[' + b",".join(cur) + b"]}")
                cur, size = [], 0
            cur.append(m)
            size += len(m) + 1
        wraps.append(b'{"type":90,"PT":37,"V":-1,"PP":[' + b",".join(cur) + b"]}")
        arena, refs = wire.pack_packets(wraps)
        refs["node"] = 100
        rounds.append((torch.from_numpy(arena.copy()).pin_memory(),
                       torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16).copy()).pin_memory(), reqs, wraps))
    n_wraps = rounds[0][1].shape[0]
    d_arena = torch.empty(max(x[0].numel() for x in rounds), dtype=torch.uint8, device="cuda")
    d_refs = torch.empty((max(x[1].shape[0] for x in rounds), 16), dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    acc = torch.empty((n, 48), dtype=torch.uint8, device="cuda")
    heads = torch.empty(n, dtype=torch.int32, device="cuda")
    ctl = torch.zeros(8, dtype=torch.int32, device="cuda")
    h_out = torch.empty(256 * n, dtype=torch.uint8).pin_memory()
    h_refs = torch.empty((2 * n, 16), dtype=torch.uint8).pin_memory()
    caps = {"json": (n, 1, 1), "req": (n, 16 * n), "enc": (256 * n, 2 * n)}

    def device_leg(r):
        a, f = rounds[r][0], rounds[r][1]
        da, dr = d_arena[: a.numel()], d_refs[: f.shape[0]]
        da.copy_(a, non_blocking=True)
        dr.copy_(f, non_blocking=True)
        j = wire.decode_json_device(ed, da, dr, caps["json"])
        d = wire.decode_json_requests_device(ed, da, dr, j.members, j.sizes[0], NOW, caps["req"])
        ctl.zero_()
        wire.propose_device_heads(ed, d.reqs, d.sizes[0], d.payload, d.sizes[1], status, acc, heads, ctl)
        enc = wire.encode_accepts_device(ed, acc, ctl.data_ptr(), d.sizes[0], heads, d.reqs, d.meta, d.sizes[0],
                                         d.payload, caps["enc"])
        caps["json"], caps["req"], caps["enc"] = j.sizes, d.sizes, enc.sizes
        h_out[: enc.sizes[0]].copy_(enc.out, non_blocking=True)
        h_refs[: enc.sizes[1]].copy_(enc.refs, non_blocking=True)
        torch.cuda.synchronize()
        return enc.sizes

    index = {names[g]: k for k, g in enumerate(gids)}

    def host_leg(r):
        mem = [m for w in rounds[r][3] for m in pj.unbatch(w)]
        reqs = np.zeros(len(mem), abi.request_dtype)
        pay = np.zeros(16 * len(mem), np.uint8)
        for k, m in enumerate(mem):
            v = m["QV"].encode(pj.CHARSET)
            reqs[k] = (gids[index[m["ID"]]], 0, m["QID"], 16 * k, len(v), m["E"], k)
            pay[16 * k: 16 * k + len(v)] = np.frombuffer(v, np.uint8)
        a, _, _ = eh.propose(reqs, pay)
        out = []
        for x in a[np.argsort(a["gid"], kind="stable")]:  # the device encoder writes in gid order
            q = rounds[r][2][index[names[int(x["gid"])]]]
            out.append(wire.encode_accept(q, int(x["slot"]), int(x["bnum"]), int(x["bcoord"]), False,
                                          int(x["median_cp"]), int(x["sender"])))
        return out

    def check(r, outs):  # each ACCEPT packet is stored once and indexed for nodes 101 and 102
        refs = h_refs[: outs["device"][1]].numpy().reshape(-1).view(abi.wire_ref_dtype)
        got = [bytes(h_out[int(x["off"]): int(x["off"]) + int(x["len"])].numpy()) for x in refs[::2]]
        assert got == outs["host"] and len(got) == n, "device and host ACCEPT packets differ"

    res = {"groups": G, "requests": n, "wrappers": int(n_wraps), "upload_bytes": int(rounds[0][0].numel())}
    if profile:
        device_leg(0)
        res["device_kernel_ms"] = min(kernel_ms(lambda: device_leg(r)) for r in range(1, reps + 1))
        res["requests_per_s_kernels"] = n / (res["device_kernel_ms"] / 1000.0)
    else:
        w = alternate({"device": device_leg, "host": host_leg}, reps + 1, check)
        for leg, s in w.items():
            res[leg] = {"wall_s_min": s, "requests_per_s_wall": n / s}
    for e in (ed, eh):
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="kernel time under torch.profiler instead of wall time")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import gigapaxos_b200
    lib = gigapaxos_b200.load_library()
    res = {"card": card_info(), "mode": "profile" if a.profile else "wall", "runs": []}
    for G in a.groups:
        run = {"groups": G}
        for name, chain in (("forward_chain", forward_chain), ("json_chain", json_chain)):
            run[name] = chain(lib, G, a.reps, a.profile)
            print(f"{name} {G}: {json.dumps(run[name])}", file=sys.stderr, flush=True)
        res["runs"].append(run)
    res["card_after"] = card_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
