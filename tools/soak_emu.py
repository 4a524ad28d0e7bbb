#!/usr/bin/env python3
"""Soak the CPU-side checks of the kernels beside the round with many random configurations (no GPU needed):

  * the kernel sources compiled for the host (tests/emu) against the oracle: k_prepare_tally, k_pause_groups,
    k_log_dir / k_log_scan / k_log_hits (as the ring lies and re-laid to wrap);
  * the oracle's phase 1b against the host-language twin (two restatements of PaxosCoordinatorState.java:264-587).

A run's sanity assertions ("some but not all groups paused", "every verdict occurred") can miss for an unlucky seed; only
mismatches between the two sides count as failures.

    python tools/soak_emu.py [iterations] [--order asc|desc|shuffle]

--order sets the order the emulated launches run their threads in (tests/emu/cuda_emu.h); shuffle draws a fresh
permutation seed for every iteration and prints it with a failure.
"""
import argparse
import ctypes as C
import os
import pathlib
import sys
import tempfile
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402

import test_log_find as tl  # noqa: E402
import test_pause_batch as tb  # noqa: E402
import test_phase1b as tp  # noqa: E402
from helpers import emu_library, oracle_library  # noqa: E402

SANITY = ("verdicts ==", "0 < want_ok.sum()", ".any()", "found >", "assert 0 < ")


class _Tmp:  # what emu_library needs of pytest's tmp_path_factory
    @staticmethod
    def mktemp(name):
        return pathlib.Path(tempfile.mkdtemp(prefix=name))


def attempt(spec, fn, *args):
    try:
        fn(*args)
        return 1
    except AssertionError:
        lines = traceback.format_exc().splitlines()
        if any(k in " ".join(lines[-4:]) for k in SANITY):
            return 0
        print(f"order {spec}:", fn.__name__, args, "\n".join(lines[-25:]))
        raise


def main(iters, order="asc"):
    lib = oracle_library()
    e1, e2, e3 = (emu_library(_Tmp, src) for src in ("p1b_emu", "pause_emu", "logfind_emu"))
    e3.emu_log_find.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                C.c_uint32, C.c_uint32]
    rng = np.random.default_rng(int(time.time()))
    ok = 0
    t0 = time.time()
    for _ in range(iters):
        spec = f"shuffle:{int(rng.integers(1 << 62))}" if order == "shuffle" else order
        for e in (e1, e2, e3):  # also restarts the launch count: an iteration's orders follow from its seed alone
            assert e.emu_set_order(spec.encode()) == 0, spec
        seed = int(rng.integers(100, 60000))
        R = int(rng.choice([1, 2, 3, 3, 4, 5]))
        wrap = bool(rng.integers(0, 2))
        ln = None
        if R >= 3 and rng.integers(0, 3) == 0:
            ln = [tp.NODES5[i] for i in rng.choice(R, size=int(rng.integers(1, R)), replace=False)]
        ok += attempt(spec, tp.test_kernel_source_on_the_host_equals_oracle, lib, e1, R, seed, wrap, int(rng.choice([1, 7, 33, 64])), ln)
        ok += attempt(spec, tp.test_oracle_phase1b_equals_the_host_twin, lib, R, seed, wrap, ln)
        ok += attempt(spec, tb.test_kernel_source_on_the_host_equals_oracle, lib, e2, int(rng.integers(0, 2)), int(rng.choice([2, 3, 5])),
                      seed, int(rng.choice([1, 33, 128])))
        ok += attempt(spec, tl.test_kernel_source_on_the_host_equals_oracle, lib, e3, seed, int(rng.choice([1, 3, 7])),
                      int(rng.choice([1, 64, 256])))
        ok += attempt(spec, tl.test_kernel_source_on_a_ring_that_wraps, lib, e3, seed)
    print(f"{iters} iterations x 5 checks, order {order}: {ok} complete, {5 * iters - ok} ended at a sanity assertion, 0 mismatches; "
          f"{time.time() - t0:.0f} s")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("iterations", type=int, nargs="?", default=50)
    ap.add_argument("--order", choices=("asc", "desc", "shuffle"), default="asc")
    a = ap.parse_args()
    main(a.iterations, a.order)
