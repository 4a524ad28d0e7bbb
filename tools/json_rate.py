#!/usr/bin/env python3
"""Rate of gpx_wire_decode_json_device on a peer's sweep: one one-slot BatchedAcceptReply per group, as JSON members of
4 MiB BATCHED_PAXOS_PACKET wrappers (how a loaded Java node sends them), at 100 K and 1 M groups.

Reports, per size: the wall-clock time of upload + call + download (median of the repeats), the kernel-only
time (torch.profiler: the sum of the device kernels of one call), and for contrast Python's json.loads plus
packets_json.parse_packet on the host over the same members.  The card, its power limit and SM clock are read in the
same run (nvidia-smi --query-gpu, read only).

    python tools/json_rate.py [--groups 100000 1000000] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.stdout else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import gigapaxos_b200
    from gigapaxos_b200 import abi, packets_json as pj, wire
    from helpers import Engine, make_config
    from wire_json_cases import wrap

    lib = gigapaxos_b200.load_library()
    lanes = [100, 101, 102]
    results = {"card_before": card(), "runs": []}
    for G in a.groups:
        e = Engine(lib, make_config(lib, max_groups=G, max_group_size=16, n_lanes=3, lane_node=lanes))
        d = np.zeros(G, abi.group_desc_dtype)
        names = ["g%d" % g for g in range(G)]
        for g in range(G):
            d[g] = (g, 0, abi.java_string_hash(names[g]), 3, [100, 101, 102] + [0] * 13, abi.INIT_BATCH)
        e.create_groups(d)
        wire.set_group_names(e, list(range(G)), names)
        # the acceptor on node 101 answers coordinator 100's ACCEPT for slot g of every group
        members = [pj.batched_accept_reply_json(names[g], 0, 101, 5, 100, g, g - 1, g, [g], [g]) for g in range(G)]
        pkts, cur, size = [], [], 0
        for m in members:
            if size + len(m) + 64 > (4 << 20):
                pkts.append(wrap(cur)[0])
                cur, size = [], 0
            cur.append(m)
            size += len(m) + 1
        if cur:
            pkts.append(wrap(cur)[0])
        arena, refs = wire.pack_packets(pkts)
        refs["node"] = 100
        h_arena = torch.from_numpy(arena.copy()).pin_memory()
        h_refs = torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16).copy()).pin_memory()
        caps = (G, G, 0)

        def chain():
            da = h_arena.to("cuda", non_blocking=True)
            dr = h_refs.to("cuda", non_blocking=True)
            out = wire.decode_json_device(e, da, dr, caps)
            return out.replies.cpu()
        rep = chain()
        got = rep.numpy().reshape(-1).view(abi.reply_dtype)
        assert len(got) == G and (got["slot"] == np.arange(G)).all()
        walls = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            chain()
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
        da, dr = h_arena.cuda(), h_refs.cuda()
        wire.decode_json_device(e, da, dr, caps)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            wire.decode_json_device(e, da, dr, caps)
            torch.cuda.synchronize()
        kern_us = sum(ev.self_device_time_total for ev in prof.key_averages()
                      if "Memcpy" not in ev.key and "Memset" not in ev.key)
        n_host = min(G, 50_000)
        w = wrap(members[:n_host])[0]
        t0 = time.perf_counter()
        pj.parse_packet(w)
        host_s = time.perf_counter() - t0
        wall = float(np.median(walls))
        r = {"groups": G, "packets": len(pkts), "bytes": int(len(arena)), "wall_ms": wall * 1e3,
             "wall_members_per_s": G / wall, "kernel_ms": kern_us / 1e3, "kernel_members_per_s": G / (kern_us * 1e-6),
             "kernel_GB_per_s": len(arena) / (kern_us * 1e-6) / 1e9,
             "host_python_members_per_s": n_host / host_s, "host_python_members": n_host}
        print(json.dumps(r))
        results["runs"].append(r)
        e.close()
        del h_arena, h_refs
    results["card_after"] = card()
    print(json.dumps({"card": results["card_after"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
