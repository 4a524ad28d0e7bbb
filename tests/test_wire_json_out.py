"""CPU: the JSON encoder's kernel source (gigapaxos_b200/csrc/gpx_wire_json_enc.cuh) compiled for the host
(tests/emu/wire_json_out_emu.cpp) against the Python model of tests/wire_json_out_cases.py: the output is byte-identical
for random worlds with hard names, 1-8 lanes, values at the int32 / int64 edges and permuted member sets; small wrapper
sizes cut often and stay within their bound; every packet parses; GPX_ERANGE writes nothing; and the JSON form decodes
(emulated gpx_wire_decode_json_device) to the records the byte form decodes to.  Also once more under AddressSanitizer
+ UBSan."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from test_wire_dev import Emu
from test_wire_json import decode_json
from wire_dev_cases import World
from wire_json_out_cases import (MAX_MEMBER, WRAP_OVERHEAD, coordinator_commit_world, expected_json, json_decisions,
                                 json_replies, json_world)

from gigapaxos_b200 import packets_json as pj, wire

NODES = [100, 101, 102, 98, 99, 97, 96, 95]  # 103 and 104 stay remote


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_json_out_emu")


def encode_json(e: Emu, rep, dec, n_dec=None, wrap=0, block=64, sizes=None):
    """emu_wire_encode_json, sized first -> (rc, rstatus_r, rstatus_d, out, refs); sizes given: one call at them"""
    rep = np.ascontiguousarray(rep if rep is not None else np.zeros(0, abi.reply_dtype))
    dec = np.ascontiguousarray(dec if dec is not None else np.zeros(0, abi.decision_dtype))
    cnt = None if n_dec is None else np.array([n_dec], np.uint32)
    rr = np.full(max(len(rep), 1), 0xAB, np.uint8)
    rd = np.full(max(len(dec), 1), 0xAB, np.uint8)
    sz = np.zeros(2, np.uint64) if sizes is None else np.array(sizes, np.uint64)

    def call(out, refs):
        return e.lib.emu_wire_encode_json(e.h, C.c_uint32(len(rep)), ptr(rep) if len(rep) else None,
                                          ptr(dec) if len(dec) else None, ptr(cnt), C.c_uint32(len(dec)), ptr(rr),
                                          ptr(rd), C.c_uint64(wrap), ptr(out), ptr(refs), ptr(sz), C.c_uint32(block))
    if sizes is not None:
        out = np.full(max(int(sz[0]), 1), 0xCD, np.uint8)
        refs = np.zeros(max(int(sz[1]), 1), abi.wire_ref_dtype)
        rc = call(out, refs)
        return rc, rr[: len(rep)], rd[: len(dec)], out, refs, sz
    rc = call(np.zeros(1, np.uint8), np.zeros(1, abi.wire_ref_dtype))
    if rc not in (0, abi.GPX_ERANGE):
        return rc, rr, rd, None, None, sz
    out = np.zeros(max(int(sz[0]), 1), np.uint8)
    refs = np.zeros(max(int(sz[1]), 1), abi.wire_ref_dtype)
    assert call(out, refs) == 0
    return 0, rr[: len(rep)], rd[: len(dec)], bytes(out[: int(sz[0])]), refs[: int(sz[1])], sz


def as_tuples(refs):
    return [(int(r["off"]), int(r["len"]), int(r["gid"]), int(r["node"])) for r in refs]


def check(e, world, named, rep, dec, n_dec=None, wrap=0, block=64):
    rc, rr, rd, out, refs, _ = encode_json(e, rep, dec, n_dec, wrap, block)
    assert rc == 0
    er, ed, eout, erefs = expected_json(world, named, rep, dec, n_dec, wrap or (4 << 20))
    assert list(rr) == list(er)
    nd = len(ed)
    assert list(rd[:nd]) == list(ed) and all(x == 0xAB for x in rd[nd:])
    assert out == eout
    assert as_tuples(refs) == erefs
    return out, refs


def world_emu(lib, world, unnamed=()):
    e = Emu(lib, world)
    if unnamed:
        e.remove(list(unnamed))
    return e, set(world.groups) - set(unnamed)


@pytest.mark.parametrize("lanes", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("seed", [1, 2])
def test_output_equals_the_model(lib, lanes, seed):
    rng = np.random.default_rng(100 * lanes + seed)
    world = json_world(rng, 40, NODES[:lanes])
    e, named = world_emu(lib, world, unnamed=list(world.groups)[:3])
    rep = json_replies(rng, world, 150, lanes)
    dec = json_decisions(rng, world, 200)
    out, refs = check(e, world, named, rep, dec, block=int(rng.choice([1, 64])))
    assert len(refs) > 10
    rst = list(encode_json(e, rep, dec)[1])
    for s in (abi.WE_SENT, abi.WE_VOID, abi.WE_NACK, abi.WE_NO_NAME) + ((abi.WE_LOCAL,) if lanes > 1 else ()):
        assert s in rst, s
    e.close()


def test_device_count_below_n_dec_max_and_empty_inputs(lib):
    rng = np.random.default_rng(7)
    world = json_world(rng, 20, NODES[:3])
    e, named = world_emu(lib, world)
    dec = json_decisions(rng, world, 80)
    check(e, world, named, None, dec, n_dec=33)
    check(e, world, named, json_replies(rng, world, 30, 3), None)
    rc, _, _, out, refs, sz = encode_json(e, None, None)
    assert rc == 0 and list(sz) == [0, 0]
    check(e, world, named, None, dec, n_dec=0)
    e.close()


def test_a_commit_to_a_replys_coordinator_shares_its_wrapper(lib):
    """permuted member sets are one recipient set, and a commit whose only remote member is the replies' coordinator
    rides in the replies' wrapper"""
    world = coordinator_commit_world([100, 101])
    e, named = world_emu(lib, world)
    rep = np.zeros(4, abi.reply_dtype)
    # group 0 [100, 103, 104] and group 1 [104, 100, 103]: acceptor 100 (lane 0) replies to coordinator 103
    rep[0] = (0, 5, 1, 103, 0, abi.who(0, 1, 0), 9)
    rep[2] = (1, 6, 1, 103, 0, abi.who(1, 2, 0), 10)
    rep[1]["who"] = rep[3]["who"] = abi.who(0, 0, abi.F_VOID)
    dec = np.zeros(2, abi.decision_dtype)
    dec[0] = (2, 7, 2, 100, 0, abi.F_DECISION, 3, 0)  # group 2 [100, 101, 103]: remote member 103 only
    dec[1] = (0, 8, 2, 100, 0, abi.F_DECISION, 1, 0)  # group 0: remote {103, 104}
    out, refs = check(e, world, named, rep, dec)
    pkts = sorted(set((int(r["off"]), int(r["len"])) for r in refs))
    assert len(pkts) == 2  # {103}: two replies and the commit of group 2; {103, 104}: the commit of group 0
    first = pj.parse_packet(out[pkts[0][0]: pkts[0][0] + pkts[0][1]])
    assert [m["kind"] for m in first["packets"]] == ["BATCHED_ACCEPT_REPLY", "BATCHED_ACCEPT_REPLY", "BATCHED_COMMIT"]
    assert as_tuples(refs)[1:] == [(pkts[1][0], pkts[1][1], 0, 103), (pkts[1][0], pkts[1][1], 0, 104)]
    e.close()


@pytest.mark.parametrize("wrap", [MAX_MEMBER + WRAP_OVERHEAD + 1, MAX_MEMBER + WRAP_OVERHEAD + 700, MAX_MEMBER + 5000])
def test_small_wrappers_cut_often_and_stay_within_bound(lib, wrap):
    rng = np.random.default_rng(wrap)
    world = json_world(rng, 12, NODES[:2], permute=False)
    e, named = world_emu(lib, world)
    rep = json_replies(rng, world, 400, 2)
    dec = json_decisions(rng, world, 400)
    out, refs = check(e, world, named, rep, dec, wrap=wrap)
    spans = sorted(set((int(r["off"]), int(r["len"])) for r in refs))
    wrappers = [out[o: o + n] for o, n in spans if out[o: o + n].startswith(b'{"type":90,"PT":37')]
    assert len(wrappers) > 20
    assert max(len(w) for w in wrappers) <= wrap
    assert sum(n for _, n in spans) == len(out)  # every packet once, nothing else
    for o, n in spans:
        d = pj.parse_packet(out[o: o + n])
        assert d["kind"] in ("ACCEPT_REPLY", "BATCHED_PAXOS_PACKET")
        if d["kind"] == "ACCEPT_REPLY":
            assert d["undigest_request"] is False
    e.close()


def test_wrap_bytes_out_of_range_and_oversized_members(lib):
    world = json_world(np.random.default_rng(3), 4, NODES[:2])
    e, _ = world_emu(lib, world)
    dec = json_decisions(np.random.default_rng(3), world, 4)
    assert encode_json(e, None, dec, wrap=MAX_MEMBER + WRAP_OVERHEAD)[0] == abi.GPX_EINVAL
    assert encode_json(e, None, dec, wrap=(4 << 20) + 1)[0] == abi.GPX_EINVAL
    # one run of 6,000 distinct 11-character slots is a BatchedCommit above GPX_JSON_MAX_MEMBER
    gid = next(g for g, (_, _, m) in world.groups.items() if any(world.lane_of(x) is None for x in m))
    big = np.zeros(6000, abi.decision_dtype)
    big["gid"], big["slot"], big["bnum"], big["bcoord"] = gid, np.arange(6000) - (1 << 31), 1, world.groups[gid][2][0]
    big["flags"] = abi.F_DECISION
    rc = encode_json(e, None, big, sizes=[1 << 24, 1 << 16])
    assert rc[0] == abi.GPX_EINVAL and (rc[3] == 0xCD).all()
    e.close()


def test_output_too_small_reports_exact_sizes_and_writes_nothing(lib):
    rng = np.random.default_rng(11)
    world = json_world(rng, 20, NODES[:3])
    e, named = world_emu(lib, world)
    rep, dec = json_replies(rng, world, 60, 3), json_decisions(rng, world, 60)
    _, _, eout, erefs = expected_json(world, named, rep, dec)
    for caps in ([0, 0], [len(eout) - 1, len(erefs)], [len(eout), len(erefs) - 1]):
        rc, _, _, out, refs, sz = encode_json(e, rep, dec, sizes=caps)
        assert rc == abi.GPX_ERANGE and list(sz) == [len(eout), len(erefs)]
        assert (out == 0xCD).all() and (refs["len"] == 0).all()
    rc, _, _, out, refs, sz = encode_json(e, rep, dec, sizes=[len(eout), len(erefs)])
    assert rc == 0 and bytes(out[: len(eout)]) == eout
    e.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_json_form_decodes_to_the_byte_forms_records(lib, seed):
    """sender lanes (100, 101, 102); the receiver serves (98, 99, 103, 104): every packet decoded at the node it is
    indexed for gives, as a multiset, the records the byte encoders' packets give"""
    rng = np.random.default_rng(seed)
    world = json_world(rng, 30, [100, 101, 102], permute=False)
    tx, named = world_emu(lib, world)
    rx = Emu(lib, World(world.groups, [98, 99, 103, 104]))
    rep = json_replies(rng, world, 120, 3)
    rep["who"] &= ~np.uint32(abi.F_NACK << 16)  # the byte form sends no NACK
    dec = json_decisions(rng, world, 150)
    _, _, _, out, refs, _ = encode_json(tx, rep, dec)
    _, bpk = tx.encode(rep, 1)
    _, bpd = tx.encode(dec, 0)
    jp = [bytes(out[int(r["off"]): int(r["off"]) + int(r["len"])]) for r in refs]
    jn = [int(r["node"]) for r in refs]
    _, mem, jrep, jdec = decode_json(rx, jp, jn)
    bst, _, _, brep, bdec = rx.decode([b for _, _, b in bpk + bpd])
    assert set(int(s) for s in mem["status"]) <= {abi.WS_OK, abi.WS_NOT_LOCAL}

    def multiset(a):
        return sorted(bytes(x.tobytes()) for x in a)
    assert multiset(jrep) == multiset(brep) and len(brep) > 20
    assert multiset(jdec) == multiset(bdec) and len(bdec) > 20
    tx.close()
    rx.close()


def test_wire_json_out_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_json_out.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
