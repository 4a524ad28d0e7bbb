"""CPU: the decisions encoder of gpx_wire_encode_decisions_device, whose record count is read on the device from
*n_ptr, as kernel source compiled for the host (tests/emu/wire_emu.cpp).  Records past the count -- valid-looking
ones in the buffer, or no memory at all -- are never encoded, never read and get no rstatus: the packets, refs and
rstatus[0:*n_ptr] equal encoding only the counted records.  Also once more under AddressSanitizer + UBSan."""
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, emu_library
from test_wire_dev import ENC_DECISIONS, Emu
from wire_dev_cases import expected_encode_decisions, random_decisions, random_world


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_emu")


def encode_counted(e: Emu, recs, count, n_max, block):
    """the device-count encoder over recs (n_max records, or only `count` of them in memory) -> (rstatus, packets)"""
    return e.encode_kind(ENC_DECISIONS, recs, n_max, count=count, block=block)


@pytest.mark.parametrize("seed", [4, 5, 6])
@pytest.mark.parametrize("block", [1, 64])
def test_decisions_past_the_device_count_are_not_encoded(emu, seed, block):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 12)
    e = Emu(emu, world)
    dec = random_decisions(rng, world, 300)
    pad = random_decisions(rng, world, 80)  # valid-looking records behind the count
    for k in (0, 1, 137, 300):
        want_rst, want = e.encode(dec[:k], 0)
        if k:
            est, exp = expected_encode_decisions(world, dec[:k])
            assert np.array_equal(want_rst, est) and want == exp
        rst, got = encode_counted(e, np.concatenate([dec[:k], pad]), k, k + len(pad), block)
        assert np.array_equal(rst[:k], want_rst) and got == want
        assert (rst[k:] == 0xAB).all()
        # a count above n_max is capped at n_max
        rst, got = encode_counted(e, dec[:k], k + 5, k, block)
        assert np.array_equal(rst[:k], want_rst) and got == want
    e.close()


def test_records_past_the_device_count_are_never_read(emu):
    """only the counted records are in memory; under AddressSanitizer any read past them traps"""
    rng = np.random.default_rng(7)
    world = random_world(rng, 12)
    e = Emu(emu, world)
    dec = random_decisions(rng, world, 200)
    for k in (0, 50, 200):
        want_rst, want = e.encode(dec[:k], 0)
        rst, got = encode_counted(e, dec[:k].copy(), k, k + 300, 64)
        assert np.array_equal(rst[:k], want_rst) and got == want and (rst[k:] == 0xAB).all()
    e.close()


def test_device_count_encoder_is_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_device.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
