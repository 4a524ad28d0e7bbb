#!/usr/bin/env python3
"""Journal garbage collection on the device (gpx_journal_compact_device) against its host model (journal.compact_files),
on journals that gpx_log_frame_device writes from cfg2-shaped rounds (3 lanes, 1-byte requests, one request per group
and round) at 100 K and 1 M groups.  Lane 0's frames of each round become one file; every other group is collected up
to its last slot and the others not at all, so half of each file's frames are unneeded and every file is compacted.  Not part of bench.py.

Reported per size (one call over all the files):
  frames, files, bytes      the input
  index_us                  gpx_journal_index over every file on the host (the walk of the length prefixes)
  call_us                   the call alone, CUDA events on its stream (kernels, sort, scans, the one synchronisation)
  kernels_us                the kernels alone, from torch.profiler in a separate pass
  wall_us                   host clock: the upload of the files from page-locked memory, the call, the download of
                            the compacted bytes into page-locked memory, and the synchronisation
  frames_per_s_*            frames / each of the above
  compact_files_frames_per_s  journal.compact_files on the first file (100 K groups only)
  frame_write_frames_per_s  gpx_log_frame_device with the download, over the same rounds, for comparison
The GPU's name, power limit and SM clocks are read in the same run.

    python tools/journal_gc_rate.py --out /tmp/journal_gc_rate.json
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from journal_rate import NODES, gpu_info  # noqa: E402

KERNELS = ("k_jgc", "k_wire_iota", "k_wire_totals", "DeviceScan", "DeviceRadixSort", "cub")


def run_size(G, rounds, reps):
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
    blobs, pos, gc, write_s, write_frames = [], [0, 0, 0], None, 0.0, 0
    pinned = torch.empty(ring, dtype=torch.uint8, pin_memory=True)
    for r in range(rounds):
        reqs, pay = make_requests_fast(gids, payload_len=1, seed=5, round_no=r)
        eng.round(reqs, pay)
        meta = np.zeros(G, abi.journal_req_dtype)
        meta["gid"], meta["req_id"], meta["entry_node"] = reqs["gid"], reqs["req_id"], reqs["entry_node"]
        meta["entry_time"] = 1760000000000 + r
        dmeta = torch.from_numpy(meta.view(np.uint8).reshape(-1, 24)).cuda()
        torch.cuda.synchronize()
        for lane in range(3):
            t0 = time.perf_counter()
            fr = eng.log_frame_device(lane, pos[lane], dmeta, G)
            n = int(fr.sizes[0])
            pinned[:n].copy_(fr.frames[:n], non_blocking=True)
            st.synchronize()
            if r > 0:
                write_s += time.perf_counter() - t0
                write_frames += int(fr.sizes[1])
            assert fr.rc == 0
            if lane == 0:
                blobs.append(pinned[:n].numpy().tobytes())
            pos[lane] = fr.from_
            eng.log_release(lane, pos[lane])
    # every other group is collected up to its last slot: half of each file's frames are unneeded
    acc = eng.dump_rows(gids, 0)["acc_slot"].astype(np.int64)
    gc = np.where(gids % 2 == 0, acc - 1, -1).astype(np.int32)
    t0 = time.perf_counter()
    file_off = np.zeros(len(blobs) + 1, np.uint32)
    file_off[1:] = np.cumsum([len(b) for b in blobs])
    starts = np.concatenate([lib.journal_index(b, int(o)) for b, o in zip(blobs, file_off[:-1])])
    index_us = (time.perf_counter() - t0) * 1e6
    n_bytes = int(file_off[-1])
    host = torch.from_numpy(np.frombuffer(b"".join(blobs), np.uint8).copy()).pin_memory()
    data = torch.empty(n_bytes, dtype=torch.uint8, device="cuda")
    d_off, d_starts = torch.from_numpy(file_off).cuda(), torch.from_numpy(starts).cuda()
    d_gc = torch.from_numpy(gc).cuda()
    back = torch.empty(n_bytes, dtype=torch.uint8, pin_memory=True)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    caps, call_us, wall_us = (0, 0), [], []
    for k in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        data.copy_(host, non_blocking=True)
        ev0.record(st)
        res = eng.journal_compact_device(data, n_bytes, d_off, d_starts, d_gc, False, caps)
        ev1.record(st)
        nb = int(res.sizes[0])
        back[:nb].copy_(res.out[:nb], non_blocking=True)
        st.synchronize()
        assert res.rc == 0
        caps = res.sizes
        if k:
            wall_us.append((time.perf_counter() - t0) * 1e6)
            call_us.append(ev0.elapsed_time(ev1) * 1e3)
    files = res.files.cpu().numpy().reshape(-1).view(abi.journal_file_dtype)
    dropped = int(files["dropped"].sum())
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = eng.journal_compact_device(data, n_bytes, d_off, d_starts, d_gc, False, caps)
        torch.cuda.synchronize()
    k_us = sum(e.device_time_total for e in prof.key_averages() if any(k in e.key for k in KERNELS))
    n = len(starts)
    out = {"groups": G, "files": len(blobs), "frames": n, "bytes": n_bytes, "dropped_frames": dropped,
           "out_bytes": int(caps[0]), "index_us": index_us, "call_us": float(np.median(call_us)),
           "wall_us": float(np.median(wall_us)), "kernels_us": k_us}
    for k in ("index", "call", "wall", "kernels"):
        out[f"frames_per_s_{k}"] = n / out[f"{k}_us"] * 1e6
    out["frame_write_frames_per_s"] = write_frames / write_s
    if G <= 100_000:
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "f0")
            with open(p, "wb") as f:
                f.write(blobs[0])
            gcl = {f"NoopPaxosApp{i}": int(gc[i]) for i in range(G)}
            t0 = time.perf_counter()
            r = journal.compact_files([p], lambda pid, ver: gcl.get(pid) if ver == 0 else None, last_readonly=False)
            t = time.perf_counter() - t0
            out["compact_files_frames_per_s"] = (r[0].kept + r[0].dropped) / t
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("journal_gc_rate measures on the GPU; none is present")
    res = {"gpu": gpu_info(), "sizes": [run_size(G, args.rounds, args.reps) for G in args.groups]}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
