#!/usr/bin/env python3
"""Journal frames on the device (gpx_log_frame_device) against the host loop they replace (journal.LogDrainer) and the
raw segment copy (gpx_log_drain_async), on cfg2-shaped rounds (3 lanes, 1-byte requests, one request per group and
round) at 100 K and 1 M groups.  Every round's segments are framed on all 3 lanes.  Not part of bench.py.

Reported per size, per lane-round (one lane's segments of one round):
  frame_call_us     the call, CUDA events on its stream around it (its kernels, CUB's scans and the one
                    synchronisation that reads the totals)
  frame_kernels_us  the kernels alone, from torch.profiler in a separate pass (k_log_dir, k_journal_meta, k_journal x2,
                    k_journal_fit, the scans, k_wire_totals)
  frame_wall_us     host clock: the call, the download of the frames into page-locked memory and the synchronisation
  frames_per_s      frames / frame_wall_us, and the same over frame_kernels_us
  bytes_per_decision   frame bytes / decided slots (one ACCEPT and one DECISION frame per slot)
  raw_copy_us       gpx_log_drain_async + gpx_log_drain_wait of the same lane's segments of a round (no frames)
  log_drainer_us    journal.LogDrainer.drain of one lane's segments of one round into an in-memory Journaler stand-in
                    (100 K groups only: one interpreted call per image)
The GPU's name, power limit and SM clocks are read in the same run.

    python tools/journal_rate.py --out /tmp/journal_rate.json
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

NODES = [100, 101, 102]
KERNELS = ("k_log_dir", "k_journal", "k_wire_totals", "DeviceScan", "cub")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.stdout else {}


class Collect:
    def __init__(self):
        self.buf = bytearray()

    def append(self, packet):
        from gigapaxos_b200 import wire
        self.buf += wire.journal_frame(packet)

    def end_batch(self):
        pass


def run_size(G, rounds, warmup, with_drainer):
    import torch
    from gigapaxos_b200 import abi, journal, load_library, wire
    from helpers import Engine, group_descs_fast, make_requests_fast
    lib = load_library()
    cfg = lib.config_defaults()
    cfg.max_groups, cfg.n_lanes, cfg.window, cfg.max_group_size = G, 3, 8, 3
    for i in range(3):
        cfg.lane_node[i] = NODES[i]
    cfg.max_batch_recs, cfg.max_batch_payload = G, 16 * G + 16
    ring = 1 << 26
    while ring < 4 * (64 + 48 * G + 16 * G + 64 + 32 * G + 64):
        ring <<= 1
    cfg.log_ring_bytes = ring
    eng = Engine(lib, cfg)
    eng.create_groups(group_descs_fast(G))
    gids = np.arange(G, dtype=np.uint32)
    wire.set_group_names(eng, gids, [f"NoopPaxosApp{i}" for i in range(G)])
    st = torch.cuda.current_stream()
    pinned = torch.empty(ring, dtype=torch.uint8, pin_memory=True)
    raw = torch.empty(ring, dtype=torch.uint8, pin_memory=True)
    pos = [0, 0, 0]
    caps = [(0, 0, 0)] * 3
    out = {"groups": G, "lane_rounds": 0, "frames": 0, "frame_bytes": 0, "decisions": 0, "frame_call_us": [],
           "frame_wall_us": [], "raw_copy_us": [], "raw_bytes": 0}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    prof_rounds = []
    for r in range(warmup + rounds + 1):
        reqs, pay = make_requests_fast(gids, payload_len=1, seed=5, round_no=r)
        eng.round(reqs, pay)
        meta = np.zeros(G, abi.journal_req_dtype)
        meta["gid"], meta["req_id"], meta["entry_node"] = reqs["gid"], reqs["req_id"], reqs["entry_node"]
        meta["entry_time"] = 1760000000000 + r
        dmeta = torch.from_numpy(meta.view(np.uint8).reshape(-1, 24)).cuda()
        torch.cuda.synchronize()
        for lane in range(3):
            t0 = time.perf_counter()
            f, nb = eng.log_drain_async(lane, raw.data_ptr(), ring)
            eng.log_drain_wait()
            t_raw = time.perf_counter() - t0
            if r == warmup + rounds:  # the last round: its kernels under the profiler, in a pass of its own
                prof_rounds.append((lane, pos[lane], dmeta, G))
                continue
            t0 = time.perf_counter()
            ev0.record(st)
            fr = eng.log_frame_device(lane, pos[lane], dmeta, G, caps[lane])
            ev1.record(st)
            n = int(fr.sizes[0])
            pinned[:n].copy_(fr.frames[:n], non_blocking=True)
            st.synchronize()
            t_wall = time.perf_counter() - t0
            assert fr.rc == 0 and fr.sizes[1] == 2 * G
            caps[lane] = fr.sizes
            if with_drainer and lane == 0 and r == warmup:
                d = journal.LogDrainer(eng, 0, Collect(), lambda g, q: (f"NoopPaxosApp{g}", 0, NODES[0],
                                                                         1760000000000 + r))
                d.offset = pos[lane]
                t0 = time.perf_counter()
                d.drain()
                out["log_drainer_us"] = (time.perf_counter() - t0) * 1e6
                assert bytes(d.j.buf) == pinned[:n].numpy().tobytes()
            pos[lane] = fr.from_
            eng.log_release(lane, pos[lane])
            if r >= warmup:
                out["lane_rounds"] += 1
                out["frames"] += int(fr.sizes[1])
                out["frame_bytes"] += n
                out["decisions"] += G
                out["frame_call_us"].append(ev0.elapsed_time(ev1) * 1e3)
                out["frame_wall_us"].append(t_wall * 1e6)
                out["raw_copy_us"].append(t_raw * 1e6)
                out["raw_bytes"] += nb
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for lane, f, dmeta, n_meta in prof_rounds:
            fr = eng.log_frame_device(lane, f, dmeta, n_meta, caps[lane])
            assert fr.rc == 0
        torch.cuda.synchronize()
    k_us = sum(e.device_time_total for e in prof.key_averages() if any(k in e.key for k in KERNELS))
    eng.close()
    med = lambda v: float(np.median(v))
    res = {"groups": G, "lane_rounds": out["lane_rounds"], "frames_per_lane_round": out["frames"] // out["lane_rounds"],
           "bytes_per_decision": out["frame_bytes"] / out["decisions"],
           "frame_call_us": med(out["frame_call_us"]), "frame_wall_us": med(out["frame_wall_us"]),
           "frame_kernels_us": k_us / len(prof_rounds), "raw_copy_us": med(out["raw_copy_us"]),
           "raw_bytes_per_lane_round": out["raw_bytes"] / out["lane_rounds"]}
    fpr = res["frames_per_lane_round"]
    res["frames_per_s_wall"] = fpr / res["frame_wall_us"] * 1e6
    res["frames_per_s_kernels"] = fpr / res["frame_kernels_us"] * 1e6
    if "log_drainer_us" in out:
        res["log_drainer_us"] = out["log_drainer_us"]
        res["log_drainer_frames_per_s"] = fpr / out["log_drainer_us"] * 1e6
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("journal_rate measures on the GPU; none is present")
    res = {"gpu": gpu_info(), "sizes": [run_size(G, args.rounds, args.warmup, G <= 100_000) for G in args.groups]}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
