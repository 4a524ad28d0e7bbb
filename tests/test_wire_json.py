"""CPU: the JSON decoder's kernel source (gigapaxos_b200/csrc/gpx_wire_json.cuh) compiled for the host
(tests/emu/wire_json_emu.cpp) with chunks of 1, 7, 16 and the product's 64 bytes, so that strings, escape runs and
members cross chunk edges: the same logical replies and commits decode to the byte decoder's records whatever their
JSON form and grouping; a malformed corpus gives what the schema model of tests/wire_json_cases.py says; the host
encoders round-trip through packets_json.parse_packet.  Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from test_wire_dev import Emu
from wire_dev_cases import random_world
from wire_json_cases import as_bytes, as_json, group_into_packets, malformed_corpus, model_batch, random_logical

from gigapaxos_b200 import packets_json as pj, wire

CHUNKS = [1, 7, 16, 64]


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    out = {ch: emu_library(tmp_path_factory, "wire_json_emu", f"GPX_JSON_CHUNK={ch}u") for ch in CHUNKS}
    for lib in out.values():
        for f in ("emu_wire_free", "emu_wire_group", "emu_wire_names", "emu_wire_names_remove", "emu_wire_names_rehash",
                  "emu_wire_decode", "emu_wire_encode", "emu_wire_decode_json"):
            getattr(lib, f).argtypes = None
    return out


def decode_json(e: Emu, pkts, nodes=None, block=64, arena_refs=None):
    arena, refs = arena_refs if arena_refs is not None else wire.pack_packets(pkts)
    if nodes is not None:
        refs["node"] = nodes
    n_bytes = len(arena)
    arena = arena if len(arena) else np.zeros(1, np.uint8)
    n = len(refs)
    status = np.full(max(n, 1), -9, np.int32)
    sizes = np.zeros(3, np.uint64)
    z = np.zeros(1, np.uint8)
    args = lambda m, r, d: (e.h, C.c_uint32(n), ptr(arena), C.c_uint64(n_bytes), ptr(refs), ptr(status), ptr(m), ptr(r),
                            ptr(d), ptr(sizes), C.c_uint32(block))
    rc = e.lib.emu_wire_decode_json(*args(z, z, z))
    assert rc in (0, abi.GPX_ERANGE), rc
    mem = np.zeros(max(int(sizes[0]), 1), abi.wire_member_dtype)
    rep = np.zeros(max(int(sizes[1]), 1), abi.reply_dtype)
    dec = np.zeros(max(int(sizes[2]), 1), abi.decision_dtype)
    assert e.lib.emu_wire_decode_json(*args(mem, rep, dec)) == 0
    return status[:n], mem[: int(sizes[0])], rep[: int(sizes[1])], dec[: int(sizes[2])]


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("vary", [False, True])
def test_json_forms_decode_as_the_byte_forms(libs, chunk, seed, vary):
    """the same logical BatchedAcceptReplies / BatchedCommits as bytes (byte decoder) and as JSON in wrappers and bare
    (JSON decoder): identical records, and each member's status is its byte packet's"""
    rng = np.random.default_rng(seed)
    world = random_world(rng, 30)
    e = Emu(libs[chunk], world)
    logical = random_logical(rng, world, 120)
    byts = [as_bytes(k, f) for k, f in logical]
    bst, _, _, brep, bdec = e.decode(byts)
    js = [as_json(k, f, rng if vary else None) for k, f in logical]
    pkts, spans = group_into_packets(rng, js)
    st, mem, rep, dec = decode_json(e, pkts, block=int(rng.choice([1, 64])))
    assert list(st) == [abi.WS_OK] * len(pkts)
    arena, refs = wire.pack_packets(pkts)
    assert [(int(m["pkt"]), int(m["off"]) - int(refs["off"][m["pkt"]]), int(m["len"])) for m in mem] == spans
    assert list(mem["status"]) == list(bst)
    assert np.array_equal(rep, brep) and np.array_equal(dec, bdec)
    assert len(rep) > 20 and len(dec) > 20
    e.close()


@pytest.mark.parametrize("chunk", CHUNKS)
def test_malformed_corpus_matches_the_schema_model(libs, chunk):
    world = random_world(np.random.default_rng(9), 30)
    e = Emu(libs[chunk], world)
    cases = malformed_corpus(world)
    pkts = [p for p, _ in cases]
    nodes = [n for _, n in cases]
    st, mem, rep, dec = decode_json(e, pkts, nodes)
    est, ems, erep, edec = model_batch(world, pkts, nodes)
    for k, (a, b) in enumerate(zip(st, est)):
        assert a == b, (k, pkts[k][:200], a, b)
    assert list(mem["status"]) == ems
    assert np.array_equal(rep, erep) and np.array_equal(dec, edec)
    # the corpus reaches every outcome
    assert {abi.WS_OK, abi.WS_MALFORMED, abi.WS_UNHANDLED} <= set(est)
    assert {abi.WS_OK, abi.WS_UNHANDLED, abi.WS_UNKNOWN_NAME, abi.WS_MALFORMED} <= set(ems)
    e.close()


@pytest.mark.parametrize("chunk", [1, 64])
def test_singleton_accept_replies_route_to_the_receiving_node(libs, chunk):
    """type 8: the destination is the node that received it (a NACK's ballot names another coordinator); QID is read as
    getInt reads it; NACK true is the host's"""
    world = random_world(np.random.default_rng(3), 20)
    e = Emu(libs[chunk], world)
    pkts, nodes = [], []
    rng = np.random.default_rng(4)
    for gid, (name, ver, members) in list(world.groups.items()):
        for node in (100, 101, 102, 98):
            q = int(rng.choice([5, (1 << 40) + 7, -(1 << 35) - 1, (1 << 31)]))
            pkts.append(pj.accept_reply_json(name, ver, members[0], 7, 103, 11, 10, q, undigest_request=bool(rng.integers(0, 5) == 0)))
            nodes.append(node)
    st, mem, rep, dec = decode_json(e, pkts, nodes)
    est, ems, erep, edec = model_batch(world, pkts, nodes)
    assert list(st) == est and list(mem["status"]) == ems
    assert np.array_equal(rep, erep) and len(dec) == 0
    assert abi.WS_NOT_LOCAL in ems and abi.WS_OK in ems and abi.WS_UNHANDLED in ems
    # (1 << 31) keeps its low 32 bits, sign-extended
    assert set(int(x) for x in rep["req_id"]) <= {5, 7, -1, -(1 << 31)}
    e.close()


def test_refs_past_the_arena_and_byte_packets(libs):
    world = random_world(np.random.default_rng(5), 4)
    e = Emu(libs[7], world)
    name, ver, members = world.groups[0]
    good = pj.batched_commit_json(name, ver, 1, members[0], 0, [1], members)
    byt = wire.encode_batched_commit(name, ver, 1, members[0], 0, [1], members)
    arena, refs = wire.pack_packets([good, byt, good])
    refs["len"][2] += 1  # one byte past the arena
    st, mem, rep, dec = decode_json(e, None, arena_refs=(arena, refs))
    assert list(st) == [abi.WS_OK, abi.WS_UNHANDLED, abi.WS_MALFORMED]
    assert len(mem) == 1
    e.close()


def test_lengths_beyond_the_arena_are_refused(libs):
    """refs may overlap, but packet lengths that add up to more than the arena (beyond the call's chunk bound) are
    GPX_EINVAL and nothing is written; overlapping refs within the bound decode as usual"""
    world = random_world(np.random.default_rng(7), 4)
    e = Emu(libs[7], world)
    name, ver, members = world.groups[0]
    good = pj.batched_commit_json(name, ver, 1, members[0], 0, [1], members)
    arena, refs = wire.pack_packets([good, b" " * len(good)])
    twice = refs.copy()
    twice[1] = twice[0]  # the same bytes twice: the lengths still add up to the arena
    st, mem, _, _ = decode_json(e, None, arena_refs=(arena, twice))
    assert list(st) == [abi.WS_OK] * 2 and len(mem) == 2
    many = np.repeat(refs[:1], 40)
    status = np.zeros(len(many), np.int32)
    sizes = np.full(3, 1 << 20, np.uint64)
    out = np.full(1 << 16, 0xAB, np.uint8)
    assert e.lib.emu_wire_decode_json(e.h, C.c_uint32(len(many)), ptr(arena), C.c_uint64(len(arena)), ptr(many),
                                      ptr(status), ptr(out), ptr(out), ptr(out), ptr(sizes), C.c_uint32(64)) == abi.GPX_EINVAL
    assert (out == 0xAB).all()
    e.close()


def test_output_too_small_reports_the_sizes(libs):
    world = random_world(np.random.default_rng(6), 10)
    e = Emu(libs[16], world)
    rng = np.random.default_rng(6)
    js = [as_json(k, f) for k, f in random_logical(rng, world, 40)]
    pkts, _ = group_into_packets(rng, js)
    arena, refs = wire.pack_packets(pkts)
    n = len(pkts)
    status = np.zeros(n, np.int32)
    sizes = np.zeros(3, np.uint64)
    z = np.zeros(1, np.uint8)
    assert e.lib.emu_wire_decode_json(e.h, C.c_uint32(n), ptr(arena), C.c_uint64(len(arena)), ptr(refs), ptr(status),
                                      ptr(z), ptr(z), ptr(z), ptr(sizes), C.c_uint32(64)) == abi.GPX_ERANGE
    assert int(sizes[0]) == 40 and int(sizes[1]) + int(sizes[2]) > 0
    e.close()


def test_host_encoders_round_trip_through_parse_packet():
    b = pj.batched_accept_reply_json("g/é", 3, 101, 7, 100, 5, 4, 9, [6, 5, 5], [1, 2, 3])
    d = pj.parse_packet(b)
    assert d["kind"] == "BATCHED_ACCEPT_REPLY" and d["paxos_id"] == "g/é" and d["version"] == 3
    assert (d["acceptor"], d["bnum"], d["bcoord"], d["slot_number"], d["max_checkpointed_slot"], d["request_id"]) == \
        (101, 7, 100, 5, 4, 9)
    assert d["slots"] == [5, 6] and d["request_ids"] == [3, 1]  # TreeMap: ascending, the last put wins
    c = pj.batched_commit_json("g", 0, -2, 101, -1, [3, 1, 3], [100, 101, 102])
    d = pj.parse_packet(c)
    assert d["kind"] == "BATCHED_COMMIT" and (d["bnum"], d["bcoord"], d["median_cp"]) == (-2, 101, -1)
    assert d["slots"] == [1, 3] and d["group"] == [100, 101, 102]
    w = pj.parse_packet(pj.batched_paxos_packet_json([b, c]))
    assert [m["kind"] for m in w["packets"]] == ["BATCHED_ACCEPT_REPLY", "BATCHED_COMMIT"]
    assert json.loads(b)["SLOTS"] == [5, 3, 6, 1]


def test_wire_json_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_json.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
