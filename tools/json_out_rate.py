#!/usr/bin/env python3
"""Rate of gpx_wire_encode_json_device on an acceptor's and a coordinator's sweep: one positive reply per group (lane 0
of 3, to a remote coordinator) and one decision per group, at 100 K and 1 M groups, beside the byte encoders
(gpx_wire_encode_replies_device + gpx_wire_encode_decisions_device) on the same records.

Reports, per size: members/s for the kernels only (torch.profiler: the sum of the device kernels of one call) and wall
(call + download of the packets, median of the repeats), and the number of messages (refs) each form produces.  The
card, its power limit and SM clock are read in the same run (nvidia-smi --query-gpu, read only).

    python tools/json_out_rate.py [--groups 100000 1000000] [--reps 5] [--out FILE]
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
    from gigapaxos_b200 import abi, wire
    from helpers import Engine, make_config

    lib = gigapaxos_b200.load_library()
    lanes = [100, 101, 102]
    results = {"card_before": card(), "runs": []}
    for G in a.groups:
        e = Engine(lib, make_config(lib, max_groups=G, max_group_size=16, n_lanes=3, lane_node=lanes))
        d = np.zeros(G, abi.group_desc_dtype)
        names = ["g%d" % g for g in range(G)]
        for g in range(G):
            d[g] = (g, 0, abi.java_string_hash(names[g]), 3, [100, 103, 104] + [0] * 13, abi.INIT_BATCH)
        e.create_groups(d)
        wire.set_group_names(e, list(range(G)), names)
        rep = np.zeros(3 * G, abi.reply_dtype)
        rep["gid"] = np.repeat(np.arange(G), 3)
        rep["who"] = abi.who(0, 0, abi.F_VOID)
        r0 = rep[0::3]
        r0["slot"], r0["bnum"], r0["bcoord"], r0["max_cp"], r0["req_id"] = np.arange(G), 5, 103, -1, np.arange(G)
        r0["who"] = abi.who(0, 1, 0)  # acceptor 100 (lane 0) -> coordinator 103
        rep[0::3] = r0
        dec = np.zeros(G, abi.decision_dtype)
        dec["gid"], dec["slot"], dec["bnum"], dec["bcoord"], dec["flags"] = np.arange(G), np.arange(G), 5, 100, abi.F_DECISION
        drep = torch.from_numpy(rep.view(np.uint8).reshape(-1, 32).copy()).cuda()
        ddec = torch.from_numpy(dec.view(np.uint8).reshape(-1, 32).copy()).cuda()
        caps = {}

        def js():
            o = wire.encode_json_device(e, drep, 3 * G, ddec, None, G, caps.get("j", (1, 1)))
            caps["j"] = o.sizes
            return o

        def byte():
            o1 = wire.encode_replies_device(e, drep, 3 * G, caps.get("r", (1, 1)))
            o2 = wire.encode_decisions_device(e, ddec, None, G, caps.get("d", (1, 1)))
            caps["r"], caps["d"] = o1.sizes, o2.sizes
            return o1, o2
        r = {"groups": G, "members": 2 * G}
        for form, fn, outs in (("json", js, lambda o: [o]), ("bytes", byte, lambda o: list(o))):
            o = fn()
            r[f"{form}_messages"] = int(sum(x.sizes[1] for x in outs(o)))
            r[f"{form}_bytes"] = int(sum(x.sizes[0] for x in outs(o)))
            walls = []
            for _ in range(a.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for x in outs(fn()):
                    x.out.cpu()
                    x.refs.cpu()
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t0)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            kern_us = sum(ev.self_device_time_total for ev in prof.key_averages()
                          if "Memcpy" not in ev.key and "Memset" not in ev.key)
            wall = float(np.median(walls))
            r[f"{form}_wall_ms"] = wall * 1e3
            r[f"{form}_wall_members_per_s"] = 2 * G / wall
            r[f"{form}_kernel_ms"] = kern_us / 1e3
            r[f"{form}_kernel_members_per_s"] = 2 * G / (kern_us * 1e-6)
        print(json.dumps(r))
        results["runs"].append(r)
        e.close()
    results["card_after"] = card()
    print(json.dumps({"card": results["card_after"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
