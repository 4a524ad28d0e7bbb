"""CPU: the forwarding kernels (gigapaxos_b200/csrc/gpx_wire_fwd.cuh: k_wire_fwd, k_json_req) compiled for the host
(tests/emu/wire_fwd_emu.cpp) beside the byte and JSON decoders they work with.

* JSON requests: seeded RequestPackets -- every QV byte raw, escaped or as \\u00XX, '/' as \\/, batched requests,
  present and absent addresses, E = -1, STOP, QF, BC, forward counts, unknown names, stale versions, digests, responses
  and receiving nodes that are not local -- as JSON members of BATCHED_PAXOS_PACKETs among reply and commit members
  decode to the requests, meta and values the byte decoder gives for their byte form, with the same statuses; a
  malformed and host-only corpus gives what the schema model says; refs past the arena, GPX_ERANGE.
* Forwards: every packet is gpx_wire_encode_request of its cut with forwardCount + 1, addressed as the restatement of
  PISM.handleProposal says, over random multi-lane worlds with locally coordinated groups, the cut rules, down
  coordinators, ping-pong, a next coordinator served by a local lane, unnamed groups and slots wrapped to -2.
Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from test_wire_dev import Emu
from wire_coord_cases import NOW_MS, random_request_packets
from wire_dev_cases import random_world
from wire_fwd_cases import expected_forwards, forward_case, json_wrappers, malformed_corpus, route, wrapper

from gigapaxos_b200 import wire


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_fwd_emu")


# ---- the decoders, on arenas ----------------------------------------------------------------------------------------
def arena_of(pkts_nodes):
    arena, refs = wire.pack_packets([p for p, _ in pkts_nodes])
    refs["node"] = [n for _, n in pkts_nodes]
    return (arena if len(arena) else np.zeros(1, np.uint8)), refs, int(refs["len"].sum())


def decode_requests(e: Emu, pkts_nodes):
    arena, refs, nb = arena_of(pkts_nodes)
    n = len(refs)
    status = np.zeros(max(n, 1), np.int32)
    sizes = np.zeros(2, np.uint64)
    z = np.zeros(16, np.uint8)
    args = lambda rq, mt, pay: (e.h, C.c_uint32(n), ptr(arena), C.c_uint64(nb), ptr(refs), C.c_int64(NOW_MS),
                                ptr(status), ptr(rq), ptr(mt), ptr(pay), ptr(sizes), C.c_uint32(64))
    assert e.lib.emu_wire_decode_requests(*args(z, z, z)) in (0, abi.GPX_ERANGE)
    reqs, meta = np.zeros(max(int(sizes[0]), 1), abi.request_dtype), np.zeros(max(int(sizes[0]), 1), abi.req_meta_dtype)
    pay = np.zeros(max(int(sizes[1]), 16), np.uint8)
    assert e.lib.emu_wire_decode_requests(*args(reqs, meta, pay)) == 0
    return status[:n], reqs[: int(sizes[0])], meta[: int(sizes[0])], pay[: int(sizes[1])]


def decode_members(e: Emu, arena, refs, nb):
    n = len(refs)
    status = np.zeros(max(n, 1), np.int32)
    sizes = np.zeros(3, np.uint64)
    z = np.zeros(1, np.uint8)
    args = lambda m, r, d: (e.h, C.c_uint32(n), ptr(arena), C.c_uint64(nb), ptr(refs), ptr(status), ptr(m), ptr(r),
                            ptr(d), ptr(sizes), C.c_uint32(64))
    assert e.lib.emu_wire_decode_json(*args(z, z, z)) in (0, abi.GPX_ERANGE)
    mem = np.zeros(max(int(sizes[0]), 1), abi.wire_member_dtype)
    rep, dec = np.zeros(max(int(sizes[1]), 1), abi.reply_dtype), np.zeros(max(int(sizes[2]), 1), abi.decision_dtype)
    assert e.lib.emu_wire_decode_json(*args(mem, rep, dec)) == 0
    return status[:n], mem[: int(sizes[0])]


def decode_json_requests(e: Emu, arena, refs, nb, mem, sizes=None, block=64):
    """(rc, status, reqs, meta, payload, sizes); sizes = the capacities (None: the sizes first)"""
    n = len(mem)
    status = np.full(max(n, 1), -9, np.int32)
    mem = mem if n else np.zeros(1, abi.wire_member_dtype)
    cap = np.array(sizes if sizes is not None else [0, 0], np.uint64)
    go = lambda cap, rq, mt, pay: e.lib.emu_wire_decode_json_requests(
        e.h, C.c_uint32(n), ptr(arena), C.c_uint64(nb), ptr(refs), C.c_uint32(len(refs)), ptr(mem), C.c_int64(NOW_MS),
        ptr(status), ptr(rq), ptr(mt), ptr(pay), ptr(cap), C.c_uint32(block))
    if sizes is None:
        z = np.zeros(16, np.uint8)
        assert go(cap, z, z, z) in (0, abi.GPX_ERANGE)
    reqs = np.zeros(max(int(cap[0]), 1), abi.request_dtype)
    meta = np.zeros(max(int(cap[0]), 1), abi.req_meta_dtype)
    pay = np.zeros(max(int(cap[1]), 16), np.uint8)
    rc = go(cap, reqs, meta, pay)
    return rc, status[:n], reqs[: int(cap[0])], meta[: int(cap[0])], pay[: int(cap[1])], cap


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("block", [1, 64])
def test_json_requests_decode_as_their_byte_form(emu, seed, block):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 40)
    e = Emu(emu, world)
    pkts = random_request_packets(rng, world, 300)
    wraps, order = json_wrappers(world, pkts, rng)
    arena, refs, nb = arena_of(wraps)
    pst, mem = decode_members(e, arena, refs, nb)
    assert (pst == abi.WS_OK).all()
    rc, st, reqs, meta, pay, _ = decode_json_requests(e, arena, refs, nb, mem, block=block)
    assert rc == 0
    # the byte form of the same requests, in member order, at the same nodes
    bst, breqs, bmeta, bpay = decode_requests(e, [(pkts[k][0], pkts[k][1]) for k, _ in order])
    req_members = [m for _, m in order]
    assert st[req_members].tolist() == bst.tolist()
    others = np.setdiff1d(np.arange(len(mem)), req_members)
    assert (st[others] == mem["status"][others]).all() and len(others) > 0
    assert {abi.WS_OK, abi.WS_UNKNOWN_NAME, abi.WS_VERSION, abi.WS_UNHANDLED, abi.WS_NOT_LOCAL} <= set(bst.tolist())
    breqs = breqs.copy()
    breqs["client"] = np.array(req_members, np.uint32)[breqs["client"]]
    assert reqs.tobytes() == breqs.tobytes() and meta.tobytes() == bmeta.tobytes() and pay.tobytes() == bpay.tobytes()
    assert len(reqs) > 300
    e.close()


def test_malformed_and_host_only_members(emu):
    rng = np.random.default_rng(9)
    world = random_world(rng, 20)
    e = Emu(emu, world)
    cases = malformed_corpus(world)
    arena, refs, nb = arena_of([(wrapper([b]), node) for b, node, _ in cases])
    pst, mem = decode_members(e, arena, refs, nb)
    assert (pst == abi.WS_OK).all() and len(mem) == len(cases)
    rc, st, reqs, _, _, _ = decode_json_requests(e, arena, refs, nb, mem)
    assert rc == 0 and st.tolist() == [c[2] for c in cases]
    assert abi.WS_MALFORMED in st.tolist() and abi.WS_UNHANDLED in st.tolist()
    # a member past the arena, and one whose packet is past the refs, are malformed; other statuses are copied
    bad = mem[-3:].copy()
    bad[0]["off"] = nb - 3
    bad[1]["pkt"] = len(refs)
    bad[2]["status"] = abi.WS_VERSION
    rc, st, _, _, _, _ = decode_json_requests(e, arena, refs, nb, bad)
    assert rc == 0 and st.tolist() == [abi.WS_MALFORMED, abi.WS_MALFORMED, abi.WS_VERSION]
    # GPX_ERANGE: the sizes, and nothing written
    rc, _, _, _, _, need = decode_json_requests(e, arena, refs, nb, mem)
    for caps in ([int(need[0]) - 1, int(need[1])], [int(need[0]), int(need[1]) - 1]):
        rc, _, reqs, _, pay, got = decode_json_requests(e, arena, refs, nb, mem, sizes=caps)
        assert rc == abi.GPX_ERANGE and got.tolist() == need.tolist()
        assert not reqs.tobytes().strip(b"\0") and not pay.tobytes().strip(b"\0")
    e.close()


# ---- forwards ----------------------------------------------------------------------------------------------------------
def encode_forwards(e: Emu, rows, reqs, meta, status, payload, down, block=64):
    emu_lib = e.lib
    acc, aux, coord = (np.ascontiguousarray(rows.acc), np.ascontiguousarray(rows.aux), np.ascontiguousarray(rows.coord))
    e._keep = (acc, aux, coord)
    emu_lib.emu_fwd_state(e.h, ptr(acc), ptr(aux), ptr(coord), C.c_int32(rows.batching), C.c_int32(rows.max_batch_size),
                          C.c_int32(rows.size_est), C.c_longlong(rows.max_batch_bytes))
    n = len(reqs)
    d = np.array(list(down) or [0], np.int32)
    rst = np.full(max(n, 1), 0xAB, np.uint8)
    sizes = np.zeros(2, np.uint64)
    z = np.zeros(16, np.uint8)
    args = lambda out, refs: (e.h, ptr(reqs), ptr(meta), C.c_uint32(n), ptr(status), ptr(payload), C.c_uint32(len(down)),
                              ptr(d), ptr(rst), ptr(out), ptr(refs), ptr(sizes), C.c_uint32(block))
    assert emu_lib.emu_wire_encode_forwards(*args(z, z)) in (0, abi.GPX_ERANGE)
    out = np.zeros(max(int(sizes[0]), 1), np.uint8)
    refs = np.zeros(max(int(sizes[1]), 1), abi.wire_ref_dtype)
    assert emu_lib.emu_wire_encode_forwards(*args(out, refs)) == 0
    return rst[:n], wire.unpack_packets(out, refs[: int(sizes[1])])


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
@pytest.mark.parametrize("cut", [dict(), dict(max_batch_size=2), dict(max_batch_bytes=40, size_est=4),
                                 dict(batching=0)])
def test_forwards_are_the_host_codec_bytes(emu, seed, cut):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 60)
    e = Emu(emu, world)
    unnamed = [g for g in world.groups if g % 4 == 0]
    e.remove(unnamed)
    named = set(world.groups) - set(unnamed)
    rows, reqs, meta, status, payload, down = forward_case(rng, world, 600, **cut)
    for dn in (down, ()):
        rst, got = encode_forwards(e, rows, reqs, meta, status, payload, dn, block=int(rng.choice([1, 64])))
        est, exp = expected_forwards(world, named, rows, reqs, meta, status, payload, dn)
        assert rst.tolist() == est.tolist()
        assert got == exp
        assert {abi.WE_SENT, abi.WE_VOID, abi.WE_ELECT, abi.WE_NO_NAME} <= set(est.tolist())
        n_sent = int((rst == abi.WE_SENT).sum())
        assert (len(got) < n_sent) if cut.get("batching", 1) else (len(got) == n_sent)
    # slots wrapped to -2 in runs this engine coordinates (or that are refused) are never forwarded
    local = [q for q in range(len(reqs)) if status[q] == abi.RS_FORWARD and
             route(world, rows, int(reqs[q]["gid"]), (int(reqs[q]["flags"]) >> 8) & 0xF)[0] != abi.RS_FORWARD]
    assert local and (rst[local] == abi.WE_VOID).all()
    e.close()


def test_forward_rules_one_by_one(emu):
    """ping-pong at forwardCount 3, the next coordinator after a down one, which is local; a coordinator that is not a
    member; an unnamed group; a wrapped slot of -2 in a group this engine coordinates"""
    from wire_dev_cases import World
    from wire_fwd_cases import Rows
    world = World({0: ("g0", 0, [100, 103, 104]), 1: ("g1", 1, [100, 103, 104]), 2: ("g2", 0, [101, 103]),
                   3: ("g3", 0, [100, 103]), 4: ("g4", 0, [100, 104]), 5: ("g5", 0, [100, 104])})
    e = Emu(emu, world)
    e.remove([4])
    rows = Rows(3, 6)
    for g, bc in ((0, 103), (1, 104), (2, 103), (3, 99), (4, 104), (5, 100)):
        rows.acc[:, g] = (0, 1, bc, 0)
    rows.coord[0, 5] = (1, 100, 0, 3)  # group 5: lane 0 (node 100) coordinates
    reqs = np.zeros(7, abi.request_dtype)
    reqs["gid"] = [0, 0, 1, 2, 3, 4, 5]
    reqs["flags"] = [0, 0, 0, 1 << 8, 0, 0, 0]
    reqs["payload_len"] = 3
    reqs["entry_node"] = 100
    meta = np.zeros(7, abi.req_meta_dtype)
    meta["forward_count"] = [3, 0, 2, 0, 0, 0, 0]
    status = np.full(7, abi.RS_FORWARD, np.int32)  # group 5's -2 is a wrapped slot
    payload = np.zeros(64, np.uint8)
    rst, got = encode_forwards(e, rows, reqs, meta, status, payload, down=[103])
    # g0: the outer request ping-pongs after the increment; g1: 104 gets forwardCount 3; g2: 103 is down, 101 after it
    # is local; g3: 99 is not a member; g4: unnamed; g5: coordinated here
    assert rst.tolist() == [abi.WE_ELECT, abi.WE_ELECT, abi.WE_SENT, abi.WE_ELECT, abi.WE_ELECT, abi.WE_NO_NAME,
                            abi.WE_VOID]
    assert [(g, n) for g, n, _ in got] == [(1, 104)]
    assert got[0][2] == wire.encode_request(wire.Request("g1", 1, 0, b"\0\0\0", entry_replica=100, forward_count=3))
    rst, got = encode_forwards(e, rows, reqs, meta, status, payload, down=[104])
    # 104 down: g1's next coordinator and g4's are node 100, a local lane; g2 goes to 103
    assert rst.tolist() == [abi.WE_ELECT, abi.WE_ELECT, abi.WE_ELECT, abi.WE_SENT, abi.WE_ELECT, abi.WE_ELECT,
                            abi.WE_VOID]
    assert [(g, n) for g, n, _ in got] == [(2, 103)]
    e.close()


def test_forward_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_forward.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
