#!/usr/bin/env python3
"""Time k_ls_settle, the sweep that writes k_round_g's lockstep records back into the per-lane planes (gpx_dev.cuh).

The engine pays it once per switch from fused rounds to another call that touches group state.  For each group count
this runs compacting rounds (every group's record VALID afterwards), then a one-group gpx_dump_rows, which settles
first, and reads the sweep's kernel time from torch.profiler.  One JSON line per group count; needs a GPU.

    python tools/settle_cost.py                 # 1M and 10M groups, 3 lanes
    python tools/settle_cost.py --groups 1000000 --reps 5
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import gigapaxos_b200  # noqa: E402
from helpers import Engine, group_descs_fast, make_config, make_requests_fast  # noqa: E402


def settle_us(G: int, reps: int) -> dict:
    lib = gigapaxos_b200.load_library()
    L = 3
    e = Engine(lib, make_config(lib, max_groups=G, n_lanes=L, window=2, max_group_size=L, max_batch_recs=G,
                                max_batch_payload=16 * G, log_ring_bytes=1 << 31))
    e.create_groups(group_descs_fast(G))
    times = []
    for r in range(reps + 1):
        reqs, pay = make_requests_fast(np.arange(G), payload_len=1, seed=3, round_no=r)
        e.round(reqs, pay, extra_cap=1)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            e.dump_rows(np.zeros(1, dtype=np.uint32), 0)
            torch.cuda.synchronize()
        ks = [k for k in prof.key_averages() if "k_ls_settle" in k.key]
        assert ks and ks[0].count == 1, "one settle sweep per switch"
        if r:  # the first sample carries the module's first-launch cost
            times.append(ks[0].device_time_total)
    e.close()
    return dict(groups=G, lanes=L, settle_us_median=statistics.median(times), settle_us=times,
                record_bytes_read=28 * G)


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--groups", type=int, nargs="*", default=[1_000_000, 10_000_000])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        print("settle_cost: no CUDA device", file=sys.stderr)
        return 1
    gpu = torch.cuda.get_device_name(0)
    for G in args.groups:
        print(json.dumps(dict(gpu=gpu, **settle_us(G, args.reps))), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
