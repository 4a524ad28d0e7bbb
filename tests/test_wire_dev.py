"""CPU: the device wire codec's kernel source (gigapaxos_b200/csrc/gpx_wire_dev.cuh) compiled for the host
(tests/emu/wire_emu.cpp) against the host codec (gpx_wire.cpp): decoding the golden vectors, seeded random packets and
malformed ones gives what gpx_wire_decode_* and the member sets say, field for field; encoding gives the bytes the host
encoders write when fed by PaxosPacketBatcher's coalescing rules (tests/wire_dev_cases.py); the name table survives
removal and rebuilds.  Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from wire_dev_cases import (World, check_decode, expected_encode_decisions, expected_encode_replies, malformed_packets,
                            random_decisions, random_packets, random_replies, random_world)

from gigapaxos_b200 import wire

GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "wire_vectors.json")))
ENC_REPLIES, ENC_DECISIONS, ENC_ACCEPTS = 0, 1, 2  # the encoders of emu_wire_encode


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_emu")


class Emu:
    """one emulated engine: the world's groups live, their names set"""

    def __init__(self, lib, world: World, G=None):
        self.lib, self.world = lib, world
        G = G or (max(world.groups) + 1)
        lanes = np.array(world.lanes, np.int32)
        self.h = C.c_void_p(lib.emu_wire_new(G, len(lanes), ptr(lanes)))
        for gid, (name, ver, members) in world.groups.items():
            m = np.array(members, np.int32)
            assert lib.emu_wire_group(self.h, C.c_uint32(gid), C.c_uint32(len(m)), ptr(m)) == 0
        self.set_names(list(world.groups))

    def set_names(self, gids):
        gids = np.array(gids, np.uint32)
        staged = np.zeros((max(len(gids), 1), 128), np.uint8)
        ver = np.zeros(max(len(gids), 1), np.int32)
        for k, g in enumerate(gids):
            name, v, _ = self.world.groups[int(g)]
            b = name.encode("iso-8859-1")
            staged[k, 0] = len(b)
            staged[k, 1: 1 + len(b)] = np.frombuffer(b, np.uint8)
            ver[k] = v
        found = np.zeros(max(len(gids), 1), np.uint32)
        self.lib.emu_wire_names(self.h, C.c_uint32(len(gids)), ptr(gids), ptr(staged), ptr(ver), ptr(found))
        return found[: len(gids)]

    def remove(self, gids):
        gids = np.array(gids, np.uint32)
        self.lib.emu_wire_names_remove(self.h, C.c_uint32(len(gids)), ptr(gids))

    def decode(self, pkts, block=64):
        arena, refs = wire.pack_packets(pkts)
        arena = arena if len(arena) else np.zeros(1, np.uint8)
        n = len(pkts)
        status = np.zeros(max(n, 1), np.int32)
        sizes = np.zeros(4, np.uint64)
        z = np.zeros(1, np.uint8)
        rc = self.lib.emu_wire_decode(self.h, C.c_uint32(n), ptr(arena), C.c_uint64(int(refs["len"].sum())), ptr(refs),
                                      ptr(status), ptr(z), ptr(z), ptr(z), ptr(z), ptr(sizes), C.c_uint32(block))
        assert rc in (0, abi.GPX_ERANGE)
        acc = np.zeros(max(int(sizes[0]), 1), abi.accept_dtype)
        blob = np.zeros(max(int(sizes[1]), 16), np.uint8)
        rep = np.zeros(max(int(sizes[2]), 1), abi.reply_dtype)
        dec = np.zeros(max(int(sizes[3]), 1), abi.decision_dtype)
        assert self.lib.emu_wire_decode(self.h, C.c_uint32(n), ptr(arena), C.c_uint64(int(refs["len"].sum())), ptr(refs),
                                        ptr(status), ptr(acc), ptr(blob), ptr(rep), ptr(dec), ptr(sizes),
                                        C.c_uint32(block)) == 0
        return status[:n], acc[: int(sizes[0])], blob[: int(sizes[1])], rep[: int(sizes[2])], dec[: int(sizes[3])]

    def encode(self, recs, is_replies, block=64):
        return self.encode_kind(ENC_REPLIES if is_replies else ENC_DECISIONS, recs, len(recs), block=block)

    def encode_kind(self, kind, recs, n_max, count=None, accepts=None, block=64):
        """emu_wire_encode over n_max records of recs, the sizes first; count = the record count the device reads (None:
        no device count), accepts = the ACCEPTs' (heads, reqs, meta, payload) -> (rstatus[n_max], packets), rstatus
        0xAB where the encoder wrote none"""
        cnt = None if count is None else np.array([count], np.uint32)
        recs = np.ascontiguousarray(recs)
        heads, reqs, meta, pay = accepts if accepts is not None else (None, None, None, None)
        heads = None if heads is None else np.ascontiguousarray(heads)
        rst = np.full(max(n_max, 1), 0xAB, np.uint8)
        sizes = np.zeros(2, np.uint64)
        z = np.zeros(16, np.uint8)
        opt = lambda a: None if a is None else ptr(a)
        r_p, h_p = (ptr(recs), opt(heads)) if len(recs) else (None, None)
        args = lambda out, refs: (self.h, C.c_int(kind), opt(cnt), C.c_uint32(n_max), r_p, h_p, opt(reqs), opt(meta),
                                  C.c_uint32(0 if reqs is None else len(reqs)), opt(pay), ptr(rst), ptr(out), ptr(refs),
                                  ptr(sizes), C.c_uint32(block))
        rc = self.lib.emu_wire_encode(*args(z, z))
        assert rc in (0, abi.GPX_ERANGE)
        out = np.zeros(max(int(sizes[0]), 1), np.uint8)
        refs = np.zeros(max(int(sizes[1]), 1), abi.wire_ref_dtype)
        rst[:] = 0xAB
        assert self.lib.emu_wire_encode(*args(out, refs)) == 0
        return rst[:n_max], wire.unpack_packets(out, refs[: int(sizes[1])])

    def close(self):
        self.lib.emu_wire_free(self.h)


GOLD_WORLD = World({0: ("NoopPaxosApp0", 0, [100, 101, 102]), 1: ("g", 0, [100, 101, 102]),
                    2: ("NoopPaxosApp12", 1, [100, 101, 102]), 3: ("pid1", 0, [23, 100, 234])})


def test_golden_vectors_decode_as_the_host_codec_says(emu):
    from test_wire import REQ1, REQ3  # noqa: the requests the golden ACCEPTs were made from
    e = Emu(emu, GOLD_WORLD)
    pkts = [bytes.fromhex(GOLD[k]["hex"]) for k in ("accept_simple", "accept_batched", "batched_accept_reply",
                                                      "batched_accept_reply_ref_main", "batched_commit",
                                                      "request_simple")]
    srcs = [("accept", REQ1), ("accept", REQ3), None, None, None, None]
    got = e.decode(pkts)
    check_decode(GOLD_WORLD, pkts, srcs, got)
    assert list(got[0]) == [abi.WS_OK, abi.WS_OK, abi.WS_OK, abi.WS_NOT_LOCAL, abi.WS_OK, abi.WS_UNHANDLED]
    assert len(got[1]) == 2 and got[1]["nreq"].tolist() == [1, 3] and len(got[3]) == 3 and len(got[4]) == 3
    e.close()


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("block", [1, 64])
def test_random_packets_decode_as_the_host_codec_says(emu, seed, block):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 40)
    e = Emu(emu, world)
    pkts, srcs = random_packets(rng, world, 300)
    check_decode(world, pkts, srcs, e.decode(pkts, block))
    e.close()


def test_malformed_unknown_and_stale_packets(emu):
    world = random_world(np.random.default_rng(9), 5)
    e = Emu(emu, world)
    cases = malformed_packets(world)
    pkts = [p for p, _ in cases]
    got = e.decode(pkts)
    assert list(got[0]) == [s for _, s in cases]
    assert len(got[1]) == len(got[3]) == len(got[4]) == 0
    e.close()


@pytest.mark.parametrize("seed", [4, 5])
def test_encoded_bytes_equal_the_host_encoders_fed_by_the_batcher_rules(emu, seed):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 12)
    e = Emu(emu, world)
    L = len(world.lanes)
    rep = random_replies(rng, world, 200, L)
    rst, got = e.encode(rep, 1)
    est, exp = expected_encode_replies(world, rep, L)
    assert np.array_equal(rst, est)
    assert got == exp and len(exp) > 10
    dec = random_decisions(rng, world, 300)
    rst, got = e.encode(dec, 0)
    est, exp = expected_encode_decisions(world, dec)
    assert np.array_equal(rst, est)
    assert got == exp and len(exp) > 10
    e.close()


def test_name_table_removal_rebuild_and_reuse(emu):
    rng = np.random.default_rng(11)
    world = random_world(rng, 300)
    e = Emu(emu, world)

    def commit(gid):
        name, ver, members = world.groups[gid]
        return wire.encode_batched_commit(name, ver, 1, members[0], 0, [1], members)
    gids = list(world.groups)
    e.remove(gids[::2])
    st = e.decode([commit(g) for g in gids])[0]
    for g, s in zip(gids, st):
        assert (s == abi.WS_UNKNOWN_NAME) == (g % 2 == 0) or s == abi.WS_NOT_LOCAL and g % 2
    # set them again: the removed cells are reused; then a rebuild drops every removed cell
    assert (e.set_names(gids[::2]) == 0xFFFFFFFF).all()
    for _ in range(3):
        e.remove(gids[1::3])
        e.set_names(gids[1::3])
    e.lib.emu_wire_names_rehash(e.h)
    st = e.decode([commit(g) for g in gids])[0]
    assert all(s in (abi.WS_OK, abi.WS_NOT_LOCAL) for s in st)
    # a name held by a gid is found under that gid
    assert e.set_names([gids[5]])[0] == gids[5]
    e.close()


def test_wire_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_dev.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
