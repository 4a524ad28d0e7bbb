"""CPU: the coordinator's wire kernels (gigapaxos_b200/csrc/gpx_wire_dev.cuh: k_wire_req_decode, k_wire_enc_keys_accepts,
k_wire_enc_accepts) compiled for the host (tests/emu/wire_emu.cpp).

* Decode: seeded REQUEST packets (singles, batched with 1-20 latched requests, empty values, every address and flag
  combination, entryReplica set and unset) give the requests and meta that the host codec's fields and
  RequestPacket.setEntryReplica say; statuses for unknown names, stale versions, digests and responses, nested batches,
  truncation and receiving nodes that are not local members.
* Encode: every packet is gpx_wire_encode_accept's bytes for the same fields -- batched slots, VOID fillers, groups
  without a name, all-local groups, bad heads, slots and ballots at the int32 wrap -- and records at and past the device
  count are neither encoded nor read.
* Round trip: k_wire_decode of the encoded ACCEPTs gives back the ACCEPT records and the blobs gpx_propose builds.
Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from test_wire_dev import ENC_ACCEPTS, Emu
from wire_coord_cases import (NOW_MS, check_requests, expected_accepts, malformed_request_packets, propose_blob,
                              random_accepts, random_request_packets)
from wire_dev_cases import random_world

from gigapaxos_b200 import wire


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_emu")


def decode_requests(e: Emu, pkts, block=64):
    """[(bytes, node, ...)] -> (status, reqs, meta, payload)"""
    arena, refs = wire.pack_packets([p[0] for p in pkts])
    refs["node"] = [p[1] for p in pkts]
    arena = arena if len(arena) else np.zeros(1, np.uint8)
    n = len(pkts)
    status = np.zeros(max(n, 1), np.int32)
    sizes = np.zeros(2, np.uint64)
    z = np.zeros(16, np.uint8)
    args = lambda rq, mt, pay: (e.h, C.c_uint32(n), ptr(arena), C.c_uint64(int(refs["len"].sum())), ptr(refs),
                                C.c_int64(NOW_MS), ptr(status), ptr(rq), ptr(mt), ptr(pay), ptr(sizes), C.c_uint32(block))
    rc = e.lib.emu_wire_decode_requests(*args(z, z, z))
    assert rc in (0, abi.GPX_ERANGE)
    reqs = np.zeros(max(int(sizes[0]), 1), abi.request_dtype)
    meta = np.zeros(max(int(sizes[0]), 1), abi.req_meta_dtype)
    pay = np.zeros(max(int(sizes[1]), 16), np.uint8)
    assert e.lib.emu_wire_decode_requests(*args(reqs, meta, pay)) == 0
    k = int(sizes[0])
    return status[:n], reqs[:k], meta[:k], pay[: int(sizes[1])]


def encode_accepts(e: Emu, acc, heads, reqs, meta, payload, count=None, block=64):
    """(rstatus[n_max], [(gid, node, bytes)]); count = the device count (None: all)"""
    return e.encode_kind(ENC_ACCEPTS, acc, len(acc), count=len(acc) if count is None else count,
                         accepts=(heads, reqs, meta, payload), block=block)


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("block", [1, 64])
def test_request_packets_decode_to_proposals(emu, seed, block):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 40)
    e = Emu(emu, world)
    pkts = random_request_packets(rng, world, 400)
    got = decode_requests(e, pkts, block)
    st = got[0]
    assert {abi.WS_OK, abi.WS_UNKNOWN_NAME, abi.WS_VERSION, abi.WS_UNHANDLED, abi.WS_NOT_LOCAL} <= set(st.tolist())
    check_requests(world, pkts, got)
    assert len(got[1]) > 400  # batched packets unrolled
    e.lib.emu_wire_free(e.h)


def test_malformed_request_packets(emu):
    rng = np.random.default_rng(9)
    world = random_world(rng, 20)
    e = Emu(emu, world)
    cases = malformed_request_packets(world)
    st, reqs, meta, _ = decode_requests(e, cases)
    assert st.tolist() == [c[2] for c in cases]
    assert len(reqs) == 1 and reqs[0]["client"] == len(cases) - 1
    e.lib.emu_wire_free(e.h)


@pytest.mark.parametrize("seed", [4, 5, 6])
@pytest.mark.parametrize("block", [1, 64])
def test_accepts_encode_to_the_host_codec_bytes(emu, seed, block):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 40)
    e = Emu(emu, world)
    unnamed = [g for g in world.groups if g % 9 == 0]
    e.remove(unnamed)
    named = set(world.groups) - set(unnamed)
    acc, heads, reqs, meta, pay = random_accepts(rng, world, 30)
    # bad heads: out of range, past the requests, at another group's request
    bad = np.nonzero((acc["flags"] & abi.F_VOID) == 0)[0][:3]
    heads = heads.copy()
    heads[bad[0]] = len(reqs) + 5
    heads[bad[1]] = len(reqs) - 1 if acc[bad[1]]["nreq"] > 1 else len(reqs) + 1
    other = np.nonzero(reqs["gid"] != acc[bad[2]]["gid"])[0]
    heads[bad[2]] = other[0]
    rst, got = encode_accepts(e, acc, heads, reqs, meta, pay, block=block)
    est, exp = expected_accepts(world, named, acc, heads, reqs, meta, pay)
    assert np.array_equal(rst, est) and got == exp
    assert {abi.WE_SENT, abi.WE_VOID, abi.WE_BAD_HEAD} <= set(rst.tolist())
    assert (acc["nreq"][rst == abi.WE_SENT] > 1).any()
    # a device count: valid-looking ACCEPTs behind it are neither encoded nor given an rstatus
    for k in (0, 1, len(acc) // 2):
        want_rst, want = expected_accepts(world, named, acc, heads, reqs, meta, pay, count=k)
        rst, got = encode_accepts(e, acc, heads, reqs, meta, pay, count=k, block=block)
        assert np.array_equal(rst[:k], want_rst) and got == want and (rst[k:] == 0xAB).all()
    e.lib.emu_wire_free(e.h)


def test_local_groups_and_no_memory_past_the_count(emu):
    """all-local groups are LOCAL; with only `count` ACCEPTs in memory, AddressSanitizer traps any read past them"""
    rng = np.random.default_rng(8)
    world = random_world(rng, 30)
    e = Emu(emu, world)
    acc, heads, reqs, meta, pay = random_accepts(rng, world, 30)
    est, exp = expected_accepts(world, set(world.groups), acc, heads, reqs, meta, pay)
    assert abi.WE_LOCAL in est.tolist()
    for k in (0, 7, len(acc)):
        want_rst, want = expected_accepts(world, set(world.groups), acc, heads, reqs, meta, pay, count=k)
        n_ptr = np.array([k], np.uint32)
        a, h = acc[:k].copy(), heads[:k].copy()
        rst = np.full(len(acc) + 50, 0xAB, np.uint8)
        sizes = np.array([1 << 24, 1 << 16], np.uint64)
        out = np.zeros(1 << 24, np.uint8)
        refs = np.zeros(1 << 16, abi.wire_ref_dtype)
        assert e.lib.emu_wire_encode(e.h, C.c_int(ENC_ACCEPTS), ptr(n_ptr), C.c_uint32(len(acc) + 50),
                                     ptr(a) if k else None, ptr(h) if k else None, ptr(reqs), ptr(meta),
                                     C.c_uint32(len(reqs)), ptr(pay), ptr(rst), ptr(out), ptr(refs), ptr(sizes),
                                     C.c_uint32(64)) == 0
        assert np.array_equal(rst[:k], want_rst) and (rst[k:] == 0xAB).all()
        assert wire.unpack_packets(out, refs[: int(sizes[1])]) == want
    e.lib.emu_wire_free(e.h)


@pytest.mark.parametrize("seed", [10, 11])
def test_encoded_accepts_decode_to_the_proposal(emu, seed):
    """the ACCEPT records and blobs k_wire_decode gives back are the ones gpx_propose builds for the requests"""
    rng = np.random.default_rng(seed)
    world = random_world(rng, 40)
    e = Emu(emu, world)
    acc, heads, reqs, meta, pay = random_accepts(rng, world, 35, entry_in_lanes=True)
    rst, got = encode_accepts(e, acc, heads, reqs, meta, pay)
    sent = [i for i in np.argsort(acc["gid"], kind="stable") if rst[i] == abi.WE_SENT]
    # one copy of each packet; only groups this engine has a lane in decode here
    seen, pkts = set(), []
    for gid, node, b in got:
        if (gid, b) not in seen:
            seen.add((gid, b))
            pkts.append((gid, b))
    assert len(pkts) == len(sent)
    keep = [(i, b) for i, (gid, b) in zip(sent, pkts) if world.lane_mask(gid)]
    assert any(acc[i]["nreq"] > 1 for i, _ in keep)
    st, dacc, blob, _, _ = e.decode([b for _, b in keep])
    assert (st == abi.WS_OK).all() and len(dacc) == len(keep)
    for (i, _), d in zip(keep, dacc):  # grouped by gid already, packet order within a gid
        for f in abi.accept_dtype.names:
            if f != "payload_off":
                assert d[f] == acc[i][f], f
        off = int(d["payload_off"])
        assert bytes(blob[off: off + int(d["payload_len"])]) == propose_blob(reqs, pay, acc[i], int(heads[i]))
    e.lib.emu_wire_free(e.h)


def test_coordinator_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_coord.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
