"""CPU: the response cache's kernels (gigapaxos_b200/csrc/gpx_respcache.cuh: k_rc_put_keys, k_rc_put, k_rc_dups,
k_rc_match, k_rc_scatter, k_rc_gen_bump) compiled for the host (tests/emu/rc_emu.cpp) against the model of
tests/rc_cases.py: the table's cells after every put, and every match's hit[], misses and count, over random cases
with keys colliding on each field, port 0 against a nonzero port, expiry exactly at the timeout, over-filled buckets,
repeated keys in one put, batched requests and gids named again between put and match.  Also once more under
AddressSanitizer + UBSan."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from rc_cases import CELLS, Cache, Names, cell_dtype, ip_word, random_case, random_keys, random_requests, rc_hash

NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = emu_library(tmp_path_factory, "rc_emu")
    lib.emu_rc_hash.restype = C.c_uint64
    lib.emu_rc_hash.argtypes = [C.c_uint32, C.c_uint32, C.c_int64, C.c_uint32, C.c_uint16]
    lib.emu_rc_cell_bytes.restype = C.c_uint32
    return lib


class EmuCache:
    """the emulated kernels over a table and name state held here"""

    def __init__(self, lib, n_buckets, T, G, names_on, block):
        self.lib, self.nb, self.T, self.G, self.block = lib, n_buckets, T, G, block
        self.cells = np.frombuffer(b"\xff" * (cell_dtype.itemsize * n_buckets * CELLS), cell_dtype).copy()
        self.gen = np.zeros(G, np.uint32)
        self.slot = np.full(G, NONE, np.uint32) if names_on else None

    def name(self, gids):
        gids = np.array(gids, np.uint32)
        if self.slot is None:
            self.slot = np.full(self.G, NONE, np.uint32)
        self.lib.emu_rc_gen_bump(ptr(self.gen), ptr(gids), C.c_uint32(len(gids)), C.c_uint32(self.block))
        self.slot[gids] = 0

    def drop(self, gids):
        self.slot[np.array(gids, np.int64)] = NONE

    def _t(self):
        return (ptr(self.cells), C.c_uint32(self.nb - 1), C.c_uint32(self.G), C.c_int64(self.T), ptr(self.gen),
                ptr(self.slot))

    def put(self, keys, now):
        keys = np.ascontiguousarray(keys)
        return self.lib.emu_rc_put(*self._t(), ptr(keys if len(keys) else np.zeros(1, abi.rc_key_dtype)),
                                   C.c_uint32(len(keys)), C.c_int64(now), C.c_uint32(self.block))

    def match(self, reqs, meta, now):
        n = len(reqs)
        hit = np.full(n, 0x55, np.int32)
        out_r = np.zeros(n, abi.request_dtype)
        out_m = np.zeros(n, abi.req_meta_dtype)
        n_out = C.c_uint32(7)
        rc = self.lib.emu_rc_match(*self._t(), ptr(np.ascontiguousarray(reqs)), ptr(np.ascontiguousarray(meta)),
                                   C.c_uint32(n), C.c_int64(now), ptr(hit), ptr(out_r), ptr(out_m), C.byref(n_out),
                                   C.c_uint32(self.block))
        assert rc == 0
        return hit, out_r[: n_out.value], out_m[: n_out.value]


def run_case(lib, case, block, G=8):
    n_buckets, T, names_on, ops = case
    names = Names(G, on=names_on)
    model = Cache(n_buckets, T, names)
    emu = EmuCache(lib, n_buckets, T, G, names_on, block)
    hits = 0
    for op in ops:
        if op[0] == "name":
            names.name(op[1])
            emu.name(op[1])
        elif op[0] == "drop":
            names.drop(op[1])
            emu.drop(op[1])
        elif op[0] == "put":
            assert emu.put(op[1], op[2]) == model.put(op[1], op[2]) == 0
            assert emu.cells.tobytes() == model.table().tobytes()
        else:
            _, reqs, meta, now = op
            hit, out_r, out_m = emu.match(reqs, meta, now)
            want, miss = model.match(reqs, meta, now)
            assert hit.tolist() == want.tolist()
            assert out_r.tobytes() == reqs[miss].tobytes() and out_m.tobytes() == meta[miss].tobytes()
            hits += int((want >= 0).sum())
    return hits


def test_hash_is_the_models(emu):
    rng = np.random.default_rng(5)
    for _ in range(500):
        gid, gen = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 32))
        req_id = int(rng.integers(-(1 << 63), (1 << 63) - 1))
        ip, port = int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 16))
        assert emu.emu_rc_hash(gid, gen, req_id, ip, port) == rc_hash(gid, gen, req_id, ip, port)
    assert emu.emu_rc_cell_bytes() == cell_dtype.itemsize
    assert ip_word((10, 1, 2, 3), 0) == 0 and ip_word((10, 1, 2, 3), 1) == 0x0A010203


@pytest.mark.parametrize("block", [1, 7, 64])
def test_kernel_source_matches_the_model_on_random_cases(emu, block):
    hits = 0
    for seed in range(40):
        hits += run_case(emu, random_case(np.random.default_rng(1000 * block + seed)), block)
    assert hits > 0


def key(gid, req_id, ip=(10, 1, 2, 3), port=4567, handle=0):
    k = np.zeros(1, abi.rc_key_dtype)
    k["gid"], k["req_id"], k["client_ip"], k["client_port"], k["handle"] = gid, req_id, ip, port, handle
    return k


def request(gid, req_id, client, ip=(10, 1, 2, 3), port=4567):
    r = np.zeros(1, abi.request_dtype)
    m = np.zeros(1, abi.req_meta_dtype)
    r["gid"], r["req_id"], r["client"] = gid, req_id, client
    m["client_ip"], m["client_port"] = ip, port
    return r, m


def cat(*pairs):
    return np.concatenate([p[0] for p in pairs]), np.concatenate([p[1] for p in pairs])


def test_expiry_ports_batches_and_generations(emu):
    e = EmuCache(emu, 1, 100, 4, True, 7)
    e.name([0, 1, 2, 3])
    assert e.put(np.concatenate([key(1, 5, handle=11), key(1, 6, port=0, handle=12)]), 1000) == 0
    # a hit until exactly the timeout
    assert e.match(*request(1, 5, 0), 1099)[0].tolist() == [11]
    assert e.match(*request(1, 5, 0), 1100)[0].tolist() == [-1]
    # port 0 equals only port 0, whatever the ip bytes say
    assert e.match(*request(1, 6, 0, ip=(9, 9, 9, 9), port=0), 1000)[0].tolist() == [12]
    assert e.match(*request(1, 6, 0, port=4567), 1000)[0].tolist() == [-1]
    assert e.match(*request(1, 5, 0, port=0), 1000)[0].tolist() == [-1]
    # two requests with one client value (a batched RequestPacket) never hit; the misses keep their order
    hit, out_r, _ = e.match(*cat(request(2, 9, 3), request(1, 5, 4), request(1, 5, 3)), 1000)
    assert hit.tolist() == [-1, 11, -1] and out_r["client"].tolist() == [3, 3]
    # named again: the old entries of gid 1 are stale; an unnamed gid never hits
    e.name([1])
    assert e.match(*request(1, 5, 0), 1000)[0].tolist() == [-1]
    assert e.put(key(1, 5, handle=13), 1000) == 0
    assert e.match(*request(1, 5, 0), 1000)[0].tolist() == [13]
    e.drop([1])
    assert e.match(*request(1, 5, 0), 1000)[0].tolist() == [-1]


def test_eviction_takes_free_then_expired_then_the_oldest(emu):
    e = EmuCache(emu, 1, 100, 4, False, 3)  # no name state: generation 0, every gid named
    for i in range(CELLS):
        assert e.put(key(0, i, handle=i), 1000 + (i % 3)) == 0
    assert e.cells["handle"].tolist() == list(range(CELLS))
    # full: the oldest put time (1000: cells 0, 3, 6), the lowest such cell
    assert e.put(key(0, 100, handle=100), 1050) == 0
    assert e.cells["handle"].tolist()[:4] == [100, 1, 2, 3]
    # cell 1 (put at 1001) has expired at 1101: it is taken before the oldest live one
    assert e.put(key(0, 101, handle=101), 1101) == 0
    assert e.cells["handle"].tolist()[:2] == [100, 101]
    # the same live key is replaced in place, in input order within one put
    assert e.put(np.concatenate([key(0, 100, handle=7), key(0, 100, handle=8)]), 1102) == 0
    assert e.cells["handle"].tolist()[:2] == [8, 101]
    assert e.match(*request(0, 100, 0), 1102)[0].tolist() == [8]


def test_bad_keys_are_einval_and_write_nothing(emu):
    e = EmuCache(emu, 4, 100, 4, True, 7)
    e.name([0, 1, 2, 3])
    assert e.put(key(0, 1, handle=1), 5) == 0
    before = e.cells.copy()
    assert e.put(np.concatenate([key(0, 2, handle=2), key(0, 3, handle=-1)]), 5) == abi.GPX_EINVAL
    assert e.put(np.concatenate([key(0, 2, handle=2), key(4, 3, handle=3)]), 5) == abi.GPX_EINVAL
    assert e.cells.tobytes() == before.tobytes()


def test_many_keys_in_few_buckets(emu):
    """a big put into a small table: each bucket's run is applied by one thread, in input order"""
    rng = np.random.default_rng(9)
    G = 64
    pool = [(int(rng.integers(G)), int(rng.integers(1 << 40)), ((10, 0, 0, i % 4), 1000 + i % 3)) for i in range(200)]
    names = Names(G, on=False)
    model = Cache(16, 1000, names)
    e = EmuCache(emu, 16, 1000, G, False, 64)
    for r in range(4):
        keys = random_keys(rng, 3000, G, pool)
        assert e.put(keys, 10 * r) == model.put(keys, 10 * r) == 0
        assert e.cells.tobytes() == model.table().tobytes()
        reqs, meta = random_requests(rng, 2000, G, pool)
        hit, out_r, out_m = e.match(reqs, meta, 10 * r + 5)
        want, miss = model.match(reqs, meta, 10 * r + 5)
        assert hit.tolist() == want.tolist() and out_r.tobytes() == reqs[miss].tobytes()


def test_response_cache_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_rc_cpu.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
