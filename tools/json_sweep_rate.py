#!/usr/bin/env python3
"""Rate of gpx_wire_encode_json_sweep_device on an entry node's whole sweep at 1 M groups of three replicas: one
request per group entering at node 100 (so the groups that nodes 103 and 104 coordinate are forwarded, one request
per cut), one positive reply per group to its ballot coordinator, and one decision per group node 100 coordinates.

Reports the number of messages (refs) the sweep sends against gpx_wire_encode_forwards_device +
gpx_wire_encode_json_device on the same records (computed from the outputs, not timed), and members/s of the sweep:
kernels only (torch.profiler: the sum of the device kernels of one call) and wall (call + download of the packets,
median of the repeats).  The card, its power limit and SM clock are read in the same run (nvidia-smi --query-gpu,
read only).

    python tools/json_sweep_rate.py [--groups 1000000] [--reps 5] [--out FILE]
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

from json_out_rate import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import gigapaxos_b200
    from gigapaxos_b200 import abi, wire
    from gigapaxos_b200.spread import coordinator_of
    from helpers import Engine, make_config, make_requests_fast

    lib = gigapaxos_b200.load_library()
    G, members = a.groups, [100, 103, 104]
    results = {"card_before": card()}
    e = Engine(lib, make_config(lib, max_groups=G, max_group_size=3, n_lanes=1, lane_node=[100], max_batch_recs=G,
                                max_batch_payload=32 * G))
    names = ["g%d" % g for g in range(G)]
    d = np.zeros(G, abi.group_desc_dtype)
    d["gid"] = np.arange(G)
    d["name_hash"] = [abi.java_string_hash(s) for s in names]
    d["n_members"] = 3
    d["members"][:, :3] = members
    d["init_mode"] = abi.INIT_BATCH
    e.create_groups(d)
    wire.set_group_names(e, list(range(G)), names)
    coord = np.array([coordinator_of(s, members) for s in names])
    # one request per group, proposed: the groups 103 and 104 coordinate are GPX_RS_FORWARD
    reqs, pay = make_requests_fast(np.arange(G), payload_len=16, seed=5, entry_lane=0, entry_node=100)
    meta = np.zeros(G, abi.req_meta_dtype)
    dreq = torch.from_numpy(reqs.view(np.uint8).reshape(-1, 32).copy()).cuda()
    dmeta = torch.from_numpy(meta.view(np.uint8).reshape(-1, 32).copy()).cuda()
    dpay = torch.from_numpy(pay.copy()).cuda()
    st = torch.empty(G, dtype=torch.int32, device="cuda")
    wire.propose_device_heads(e, dreq, G, dpay, len(pay), st, torch.empty((G, 48), dtype=torch.uint8, device="cuda"),
                              torch.empty(G, dtype=torch.int32, device="cuda"),
                              torch.zeros(8, dtype=torch.int32, device="cuda"))
    # a round's replies (acceptor 100 to each group's coordinator) and commits (of the groups 100 coordinates)
    rep = np.zeros(G, abi.reply_dtype)
    rep["gid"], rep["slot"], rep["bnum"], rep["bcoord"], rep["max_cp"] = np.arange(G), 7, 0, coord, -1
    rep["req_id"] = np.arange(G)
    rep["who"] = [abi.who(0, members.index(int(c)), 0 if c != 100 else abi.F_VOID) for c in coord]
    own = np.nonzero(coord == 100)[0]
    dec = np.zeros(len(own), abi.decision_dtype)
    dec["gid"], dec["slot"], dec["bnum"], dec["bcoord"], dec["flags"] = own, 7, 0, 100, abi.F_DECISION
    drep = torch.from_numpy(rep.view(np.uint8).reshape(-1, 32).copy()).cuda()
    ddec = torch.from_numpy(dec.view(np.uint8).reshape(-1, 32).copy()).cuda()
    caps = {}

    def sweep():
        o = wire.encode_json_sweep_device(e, drep, G, ddec, None, len(dec), dreq, dmeta, G, st, dpay, [],
                                          caps.get("s", (1, 1)))
        caps["s"] = o.sizes
        return [o]

    def apart():
        o1 = wire.encode_forwards_device(e, dreq, dmeta, G, st, dpay, [], caps.get("f", (1, 1)))
        o2 = wire.encode_json_device(e, drep, G, ddec, None, len(dec), caps.get("j", (1, 1)))
        caps["f"], caps["j"] = o1.sizes, o2.sizes
        return [o1, o2]

    o = sweep()[0]
    n_fwd = int((o.rstatus_reqs == abi.WE_SENT).sum().item())
    n_members = int((o.rstatus_replies == abi.WE_SENT).sum().item()) + len(dec) + n_fwd
    r = {"groups": G, "replicas": 3, "forwards": n_fwd, "members": n_members}
    for form, fn in (("sweep", sweep), ("forwards_plus_json", apart)):
        outs = fn()
        r[f"{form}_messages"] = int(sum(x.sizes[1] for x in outs))
        r[f"{form}_bytes"] = int(sum(x.sizes[0] for x in outs))
        walls = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for x in fn():
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
        r[f"{form}_wall_members_per_s"] = n_members / wall
        r[f"{form}_kernel_ms"] = kern_us / 1e3
        r[f"{form}_kernel_members_per_s"] = n_members / (kern_us * 1e-6)
    print(json.dumps(r))
    results["run"] = r
    e.close()
    results["card_after"] = card()
    print(json.dumps({"card": results["card_after"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
