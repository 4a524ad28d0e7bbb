#!/usr/bin/env python3
"""Rates of the response cache (gpx_response_cache_put_device / _match_device) on the device.

* put_match -- a table of 2^20 buckets (8 cells each, 320 MiB); 1 M requests with distinct client values, of which
  0 %, 1 % or 50 % have a live entry.  `put` is the time of one call putting 1 M fresh keys into the table, `match` of
  one call over the 1 M requests.  Each is the median and the best of --reps calls, timed by CUDA events around the
  call on torch's stream (each call ends in its one synchronisation), after a warm-up call.  The hit count is checked.
* chain -- what match adds to a coordinator's decode -> propose: one client REQUEST per group (groups {100, 101, 102},
  node 100 coordinates every group) decoded by gpx_wire_decode_requests_device and proposed by
  gpx_propose_device_heads, with and without gpx_response_cache_match_device between them (an empty table: every
  request is a miss and is proposed as before).  The two legs run on two engines in the same state, alternately, and
  must give the same statuses; CUDA events time each leg from the decode's start to the proposal's end.

The card's name, power limit and SM clock are read in the same run (nvidia-smi --query-gpu, read only).

    python tools/rc_rate.py [--requests 1000000] [--groups 100000 1000000] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from wire_rate import card_info  # noqa: E402

NOW = 1_700_000_000_000
BUCKETS = 1 << 20
TIMEOUT_MS = 10_000  # REQUEST_TIMEOUT, PaxosConfig


def timed(fn):
    """ms of fn() between two CUDA events on torch's current stream"""
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def stats(ms):
    return {"median_ms": round(float(np.median(ms)), 4), "best_ms": round(float(min(ms)), 4)}


def put_match(lib, N, reps):
    import torch
    from gigapaxos_b200 import abi
    from helpers import Engine, make_config
    G = N
    e = Engine(lib, make_config(lib, max_groups=G, n_lanes=1, lane_node=[100], max_batch_recs=1024,
                                log_ring_bytes=1 << 20))
    rng = np.random.default_rng(1)
    reqs = np.zeros(N, abi.request_dtype)
    reqs["gid"] = np.arange(N) % G
    reqs["req_id"] = rng.integers(0, 1 << 62, size=N)
    reqs["client"] = np.arange(N)
    meta = np.zeros(N, abi.req_meta_dtype)
    meta["client_ip"] = [10, 1, 2, 3]
    meta["client_port"] = 4567
    d_reqs = torch.from_numpy(reqs.view(np.uint8).reshape(N, 32)).cuda()
    d_meta = torch.from_numpy(meta.view(np.uint8).reshape(N, 32)).cuda()
    hit = torch.empty(N, dtype=torch.int32, device="cuda")
    out_r = torch.empty((N, 32), dtype=torch.uint8, device="cuda")
    out_m = torch.empty((N, 32), dtype=torch.uint8, device="cuda")

    def keys_of(idx, handle0):
        k = np.zeros(len(idx), abi.rc_key_dtype)
        k["gid"], k["req_id"] = reqs["gid"][idx], reqs["req_id"][idx]
        k["client_ip"], k["client_port"] = [10, 1, 2, 3], 4567
        k["handle"] = handle0 + np.arange(len(idx))
        return torch.from_numpy(k.view(np.uint8).reshape(len(idx), 24)).cuda()

    out = {"requests": N, "buckets": BUCKETS}
    # put: 1 M fresh keys (other req_ids than the requests'), into a table cleared before each call
    fresh = np.zeros(N, abi.rc_key_dtype)
    fresh["gid"], fresh["req_id"], fresh["handle"] = reqs["gid"], reqs["req_id"] ^ (1 << 62), np.arange(N)
    fresh["client_ip"], fresh["client_port"] = [10, 1, 2, 3], 4567
    d_fresh = torch.from_numpy(fresh.view(np.uint8).reshape(N, 24)).cuda()
    ms = []
    for r in range(reps + 1):
        e.response_cache_init(BUCKETS, TIMEOUT_MS)
        t, _ = timed(lambda: e.response_cache_put(d_fresh, N, NOW))
        if r:
            ms.append(t)
    out["put"] = stats(ms)
    out["put"]["Mkeys_per_s"] = round(N / (out["put"]["median_ms"] * 1e3), 1)
    for frac in (0.0, 0.01, 0.5):
        e.response_cache_init(BUCKETS, TIMEOUT_MS)
        idx = rng.permutation(N)[: int(frac * N)]
        if len(idx):
            e.response_cache_put(keys_of(idx, 0), len(idx), NOW)
        ms, n_out = [], None
        for r in range(reps + 1):
            t, n_out = timed(lambda: e.response_cache_match(d_reqs, d_meta, N, NOW + 1, hit, out_r, out_m))
            if r:
                ms.append(t)
        assert n_out == N - len(idx), (n_out, N, len(idx))
        s = stats(ms)
        s["Mreq_per_s"] = round(N / (s["median_ms"] * 1e3), 1)
        out[f"match_{int(frac * 100)}pct"] = s
    e.close()
    return out


def chain(lib, G, reps):
    import torch
    from gigapaxos_b200 import wire
    from helpers import Engine, group_descs_fast, make_config
    from test_wire_coord_gpu import request_arena
    names = [f"NoopPaxosApp{i}" for i in range(G)]
    gids = np.arange(G, dtype=np.uint32)
    legs = {}
    for leg in ("plain", "match"):
        e = Engine(lib, make_config(lib, max_groups=G, n_lanes=1, lane_node=[100], window=8, max_batch_recs=G,
                                    max_batch_payload=16 * G, log_ring_bytes=1 << 20))
        e.create_groups(group_descs_fast(G, members=(100, 101, 102)))
        wire.set_group_names(e, gids, names)
        if leg == "match":
            e.response_cache_init(BUCKETS, TIMEOUT_MS)
        legs[leg] = e
    arena, refs = request_arena([(wire.encode_request(wire.Request(names[i], 0, i + 1, b"12345678",
                                                                   client=("10.1.2.3", 4567))), 100)
                                 for i in range(G)])
    st = {k: torch.empty(G, dtype=torch.int32, device="cuda") for k in legs}
    acc = torch.empty((G, 48), dtype=torch.uint8, device="cuda")
    heads = torch.empty(G, dtype=torch.int32, device="cuda")
    hit = torch.empty(G, dtype=torch.int32, device="cuda")
    out_r = torch.empty((G, 32), dtype=torch.uint8, device="cuda")
    out_m = torch.empty((G, 32), dtype=torch.uint8, device="cuda")

    def run(leg):
        e = legs[leg]
        d = wire.decode_requests_device(e, arena, refs, NOW, (G, 16 * G))
        reqs, n = d.reqs, d.sizes[0]
        if leg == "match":
            n = e.response_cache_match(d.reqs, d.meta, n, NOW, hit, out_r, out_m)
            reqs = out_r
        ctl = torch.zeros(8, dtype=torch.int32, device="cuda")
        wire.propose_device_heads(e, reqs, n, d.payload, d.sizes[1], st[leg], acc, heads, ctl)
        return n

    ms = {k: [] for k in legs}
    for r in range(reps + 1):  # round 0 warms up; window 8 holds every round's proposal
        ns = {}
        for leg in legs:
            t, ns[leg] = timed(lambda: run(leg))
            if r:
                ms[leg].append(t)
        assert ns["plain"] == ns["match"] == G
        assert torch.equal(st["plain"], st["match"])
    out = {"groups": G, "decode_propose": stats(ms["plain"]), "decode_match_propose": stats(ms["match"])}
    out["match_adds_ms"] = round(out["decode_match_propose"]["median_ms"] - out["decode_propose"]["median_ms"], 4)
    for e in legs.values():
        e.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=1_000_000)
    ap.add_argument("--groups", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert a.reps <= 7, "the chain's engines hold 8 proposals per group (window 8)"
    import gigapaxos_b200
    lib = gigapaxos_b200.load_library()
    res = {"card": card_info(), "put_match": put_match(lib, a.requests, a.reps)}
    print(f"put_match: {json.dumps(res['put_match'])}", file=sys.stderr, flush=True)
    res["chain"] = []
    for G in a.groups:
        res["chain"].append(chain(lib, G, a.reps))
        print(f"chain {G}: {json.dumps(res['chain'][-1])}", file=sys.stderr, flush=True)
    res["card_after"] = card_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
