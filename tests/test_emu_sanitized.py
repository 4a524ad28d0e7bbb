"""The emulated CUDA kernels (tests/emu: k_prepare_tally, k_pause_groups, k_select_groups, k_log_dir / k_log_scan /
k_log_hits compiled for the host) once more under AddressSanitizer + UBSan: every buffer numpy hands them and every local
array of theirs gets red zones, signed overflow and misaligned access trap.  The sanitizer runtime has to be the first
library of the process, hence the child pytest."""
import os
import subprocess
import sys

import pytest

from helpers import ROOT


def test_emulated_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_phase1b.py"), os.path.join(ROOT, "tests", "test_pause_batch.py"),
                        os.path.join(ROOT, "tests", "test_log_find.py"),
                        "-k", "kernel_source or run_away or absurd or more_segments or select_kernel or missing_kernel"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
