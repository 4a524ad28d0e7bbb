"""CPU: the sweep encoder's kernel source (gigapaxos_b200/csrc/gpx_wire_json_enc.cuh with gpx_wire_fwd.cuh's walk)
compiled for the host (tests/emu/wire_json_sweep_emu.cpp) against the Python model of tests/wire_json_sweep_cases.py:
byte-identical output for random worlds of 1-8 lanes at block sizes 1, 7 and 64, with hard names and values; the
forwards' statuses and lone packets are the forwards encoder's (tests/emu/wire_fwd_emu.cpp); with no requests the
output is the JSON-out call's; a forward rides in the wrapper of its lane's replies to the same coordinator; an
oversized value goes alone; GPX_ERANGE writes nothing; and the sweep decodes (JSON decoders and the byte requests
decoder) to the requests the byte forwards decode to.  Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from test_wire_dev import Emu
from test_wire_forward import decode_json_requests, decode_members, decode_requests, encode_forwards, arena_of
from test_wire_json_out import NODES, as_tuples, encode_json
from wire_dev_cases import World
from wire_fwd_cases import Rows, expected_forwards, forward_case
from wire_json_out_cases import MAX_MEMBER, WRAP_OVERHEAD, json_decisions, json_replies, json_world
from wire_json_sweep_cases import coordinator_world, expected_sweep, forward_cuts, forward_member, forward_packet

from gigapaxos_b200 import packets_json as pj, wire


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_json_sweep_emu")


@pytest.fixture(scope="module")
def fwd_lib(tmp_path_factory):
    """the forwards encoder and the requests decoders, for the comparisons"""
    return emu_library(tmp_path_factory, "wire_fwd_emu")


def set_rows(e: Emu, rows: Rows):
    acc, aux, coord = (np.ascontiguousarray(rows.acc), np.ascontiguousarray(rows.aux), np.ascontiguousarray(rows.coord))
    e._keep = (acc, aux, coord)
    e.lib.emu_fwd_state(e.h, ptr(acc), ptr(aux), ptr(coord), C.c_int32(rows.batching), C.c_int32(rows.max_batch_size),
                        C.c_int32(rows.size_est), C.c_longlong(rows.max_batch_bytes))


def sweep(e: Emu, rep, dec, fwd=None, n_dec=None, wrap=0, block=64, sizes=None):
    """emu_wire_encode_json_sweep, sized first -> (rc, rstatus_r, rstatus_d, rstatus_q, out, refs, sizes); fwd = (rows,
    reqs, meta, status, payload, down) or None; sizes given: one call at them"""
    rep = np.ascontiguousarray(rep if rep is not None else np.zeros(0, abi.reply_dtype))
    dec = np.ascontiguousarray(dec if dec is not None else np.zeros(0, abi.decision_dtype))
    cnt = None if n_dec is None else np.array([n_dec], np.uint32)
    if fwd is None:
        reqs, meta, status, payload, down = (np.zeros(0, abi.request_dtype), np.zeros(0, abi.req_meta_dtype),
                                             np.zeros(1, np.int32), np.zeros(16, np.uint8), ())
    else:
        rows, reqs, meta, status, payload, down = fwd
        set_rows(e, rows)
    nq = len(reqs)
    d = np.array(list(down) or [0], np.int32)
    rr = np.full(max(len(rep), 1), 0xAB, np.uint8)
    rd = np.full(max(len(dec), 1), 0xAB, np.uint8)
    rq = np.full(max(nq, 1), 0xAB, np.uint8)
    sz = np.zeros(2, np.uint64) if sizes is None else np.array(sizes, np.uint64)

    def call(out, refs):
        return e.lib.emu_wire_encode_json_sweep(
            e.h, C.c_uint32(len(rep)), ptr(rep) if len(rep) else None, ptr(dec) if len(dec) else None, ptr(cnt),
            C.c_uint32(len(dec)), ptr(reqs) if nq else None, ptr(meta) if nq else None, C.c_uint32(nq), ptr(status),
            ptr(payload), C.c_uint32(len(down)), ptr(d), ptr(rr), ptr(rd), ptr(rq), C.c_uint64(wrap), ptr(out),
            ptr(refs), ptr(sz), C.c_uint32(block))
    if sizes is not None:
        out = np.full(max(int(sz[0]), 1), 0xCD, np.uint8)
        refs = np.zeros(max(int(sz[1]), 1), abi.wire_ref_dtype)
        rc = call(out, refs)
        return rc, rr[: len(rep)], rd[: len(dec)], rq[:nq], out, refs, sz
    rc = call(np.zeros(1, np.uint8), np.zeros(1, abi.wire_ref_dtype))
    if rc not in (0, abi.GPX_ERANGE):
        return rc, rr, rd, rq, None, None, sz
    out = np.zeros(max(int(sz[0]), 1), np.uint8)
    refs = np.zeros(max(int(sz[1]), 1), abi.wire_ref_dtype)
    assert call(out, refs) == 0
    return 0, rr[: len(rep)], rd[: len(dec)], rq[:nq], bytes(out[: int(sz[0])]), refs[: int(sz[1])], sz


def check(e, world, named, rep, dec, fwd, n_dec=None, wrap=0, block=64):
    rc, rr, rd, rq, out, refs, _ = sweep(e, rep, dec, fwd, n_dec, wrap, block)
    assert rc == 0
    er, ed, eq, eout, erefs, lone = expected_sweep(world, named, rep, dec, fwd, n_dec, wrap or (4 << 20))
    assert list(rr) == list(er)
    nd = len(ed)
    assert list(rd[:nd]) == list(ed) and all(x == 0xAB for x in rd[nd:])
    assert list(rq) == list(eq)
    assert out == eout
    assert as_tuples(refs) == erefs
    return out, refs, lone


def world_emu(lib, world, unnamed=()):
    e = Emu(lib, world)
    if unnamed:
        e.remove(list(unnamed))
    return e, set(world.groups) - set(unnamed)


def edge_values(rng, reqs, meta):
    """int32 / int64 edges of ET, QID and the forward count on some requests"""
    i64 = [-(1 << 63), (1 << 63) - 1, -1, 0]
    for q in range(len(reqs)):
        if rng.integers(0, 4) == 0:
            reqs[q]["req_id"] = int(rng.choice(i64))
        if rng.integers(0, 4) == 0:
            meta[q]["entry_time"] = int(rng.choice(i64))
        if rng.integers(0, 6) == 0:
            meta[q]["forward_count"] = int(rng.choice([-(1 << 31), (1 << 31) - 1, -2, 2]))


def random_case(rng, lanes, n_groups=40, n_req=300, **cut):
    world = json_world(rng, n_groups, NODES[:lanes])
    rows, reqs, meta, status, payload, down = forward_case(rng, world, n_req, L=lanes, **cut)
    edge_values(rng, reqs, meta)
    return world, (rows, reqs, meta, status, payload, down)


@pytest.mark.parametrize("lanes", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("block", [1, 7, 64])
def test_output_equals_the_model_and_the_forwards_encoder(lib, fwd_lib, lanes, block):
    rng = np.random.default_rng(10 * lanes + block)
    world, fwd = random_case(rng, lanes, n_groups=150, **([dict(max_batch_size=2), dict()][block % 2]))
    unnamed = [g for g in world.groups if g % 8 == 0]
    e, named = world_emu(lib, world, unnamed)
    rep = json_replies(rng, world, 120, lanes)
    dec = json_decisions(rng, world, 150)
    out, refs, lone = check(e, world, named, rep, dec, fwd, block=block)
    rows, reqs, meta, status, payload, down = fwd
    # the statuses, and the lone packets, are the forwards encoder's
    f = Emu(fwd_lib, world)
    f.remove(unnamed)
    frst, fpk = encode_forwards(f, rows, reqs, meta, status, payload, down, block=block)
    rq = sweep(e, rep, dec, fwd, block=block)[3]
    assert frst.tolist() == rq.tolist()
    assert frst.tolist() == expected_forwards(world, named, rows, reqs, meta, status, payload, down)[0].tolist()
    # the lone packets follow the bare NACKs: each is the forwards encoder's packet for its cut, with its ref
    n_nack = sum(1 for r in refs if out[int(r["off"]): int(r["off"]) + 20].startswith(b'{"type":90,"PT":8,'))
    lone_pk = [(int(r["gid"]), int(r["node"]), out[int(r["off"]): int(r["off"]) + int(r["len"])])
               for r in refs[n_nack: n_nack + len(lone)]]
    _, cuts = forward_cuts(world, named, rows, reqs, meta, status, down)
    assert len(cuts) == len(fpk)
    assert lone_pk == [p for (k, b, _, _, _), p in zip(cuts, fpk) if (k, b) in lone]
    assert any(b - k > 1 for k, b in lone)
    st = set(rq.tolist())
    assert {abi.WE_SENT, abi.WE_VOID, abi.WE_ELECT, abi.WE_NO_NAME} <= st
    wrapped = [m for p in pkts_of(out, refs) if p.startswith(b'{"type":90,"PT":37') for m in members_of(p)]
    assert sum(1 for m in wrapped if m["PT"] == pj.PT_REQUEST) > 5
    e.close()
    f.close()


def members_of(wrapper):
    return json.loads(wrapper.decode("iso-8859-1"))["PP"]


def pkts_of(out, refs):
    return [out[o: o + n] for o, n in sorted(set((int(r["off"]), int(r["len"])) for r in refs))]


def test_no_requests_is_the_json_out_call(lib):
    rng = np.random.default_rng(5)
    for lanes in (1, 3, 8):
        world = json_world(rng, 30, NODES[:lanes])
        e, named = world_emu(lib, world, list(world.groups)[:2])
        rep, dec = json_replies(rng, world, 100, lanes), json_decisions(rng, world, 120)
        for n_dec, wrap in ((None, 0), (40, MAX_MEMBER + WRAP_OVERHEAD + 900), (0, 0)):
            a = sweep(e, rep, dec, None, n_dec, wrap)
            b = encode_json(e, rep, dec, n_dec, wrap)
            assert a[0] == b[0] == 0
            assert a[1].tolist() == b[1].tolist() and a[2].tolist() == b[2].tolist() and a[3].size == 0
            assert a[4] == b[3] and a[5].tobytes() == b[4].tobytes() and a[6].tolist() == b[5].tolist()
        assert sweep(e, None, None)[6].tolist() == [0, 0]
        for caps in ([0, 0], [10, 1]):
            a, b = sweep(e, rep, dec, sizes=caps), encode_json(e, rep, dec, sizes=caps)
            assert a[0] == b[0] == abi.GPX_ERANGE and a[6].tolist() == b[5].tolist()
        e.close()


def coordinator_case():
    """lane 0 (node 100) replies to coordinator 103 and forwards one request of each group to it"""
    world = coordinator_world()
    rows = Rows(3, 3)
    for g, bc in ((0, 103), (1, 103), (2, 104)):
        rows.acc[:, g] = (0, 1, bc, 0)
    reqs = np.zeros(4, abi.request_dtype)
    reqs["gid"] = [0, 1, 1, 2]
    reqs["req_id"] = [11, 12, 13, 14]
    reqs["payload_off"] = [0, 16, 32, 48]
    reqs["payload_len"] = [3, 2, 0, 5]
    reqs["entry_node"] = 100
    meta = np.zeros(4, abi.req_meta_dtype)
    meta[0] = wire.req_meta(wire.Request("x", 0, 0, b"", client=("10.0.0.1", 2000), should_return=True,
                                         forward_count=1, entry_time=77))
    payload = np.frombuffer(b'a"\\' + bytes(13) + b"\x7f\xe9" + bytes(14) + bytes(16) + b"\x00\x1fxyz" + bytes(11),
                            np.uint8).copy()
    status = np.full(4, abi.RS_FORWARD, np.int32)
    rep = np.zeros(6, abi.reply_dtype)
    rep[0] = (0, 5, 1, 103, 0, abi.who(0, 1, 0), 9)  # group 0 [100, 103]: lane 0 -> 103
    rep[3] = (1, 6, 1, 103, 0, abi.who(0, 2, 0), 10)  # group 1 [100, 101, 103]: lane 0 -> 103
    rep[4] = (1, 6, 1, 103, 0, abi.who(1, 2, 0), 10)  # lane 1 (101) -> 103
    for i in (1, 2, 5):
        rep[i]["who"] = abi.who(0, 0, abi.F_VOID)
    return world, rows, reqs, meta, status, payload, rep


@pytest.mark.parametrize("max_batch_size", [1, 5])
def test_a_forward_shares_the_wrapper_of_its_lanes_replies_to_the_coordinator(lib, max_batch_size):
    world, rows, reqs, meta, status, payload, rep = coordinator_case()
    rows.max_batch_size = max_batch_size
    e, named = world_emu(lib, world)
    fwd = (rows, reqs, meta, status, payload, ())
    out, refs, lone = check(e, world, named, rep, None, fwd)
    pk = pkts_of(out, refs)
    t = as_tuples(refs)
    if max_batch_size == 1:  # every cut one request: all members
        assert lone == []
        assert [(g, n) for _, _, g, n in t] == [(0, 103), (0, 104), (1, 103)]
        kinds = [m["PT"] for m in members_of(out[t[0][0]: t[0][0] + t[0][1]])]
        assert kinds == [34, 34, 1, 1, 1]
        assert forward_member(world, reqs, meta, payload, 0) in out
    else:  # group 1's two requests are one cut with a batched request: alone, first
        assert lone == [(1, 3)]
        assert [(g, n) for _, _, g, n in t] == [(1, 103), (0, 103), (0, 104), (1, 103)]
        assert pk[0] == forward_packet(world, reqs, meta, payload, 1, 3)
        kinds = [m["PT"] for m in members_of(out[t[1][0]: t[1][0] + t[1][1]])]
        assert kinds == [34, 34, 1]
    e.close()


def test_an_oversized_value_is_sent_alone(lib, fwd_lib):
    world = World({0: ("big", 0, [100, 103]), 1: ("mid", 0, [100, 103]), 2: ("esc", 0, [100, 103])}, [100])
    rows = Rows(1, 3, batching=0)
    rows.acc[0, :] = (0, 1, 103, 0)
    vals = [b"a" * 70000, b"b" * 20000, b"\x01" * 12000]
    reqs = np.zeros(3, abi.request_dtype)
    reqs["gid"] = [0, 1, 2]
    reqs["payload_off"] = [0, 70000, 90000]
    reqs["payload_len"] = [len(v) for v in vals]
    payload = np.frombuffer(b"".join(vals) + bytes(16), np.uint8).copy()
    meta = np.zeros(3, abi.req_meta_dtype)
    status = np.full(3, abi.RS_FORWARD, np.int32)
    e, named = world_emu(lib, world)
    fwd = (rows, reqs, meta, status, payload, ())
    out, refs, lone = check(e, world, named, None, None, fwd)
    assert lone == [(0, 1), (2, 3)]  # 70,000 bytes, and 12,000 bytes escaped six-fold; 20,000 bytes fit
    f = Emu(fwd_lib, world)
    _, fpk = encode_forwards(f, rows, reqs, meta, status, payload, ())
    t = as_tuples(refs)
    assert [out[o: o + n] for o, n, _, _ in t[:2]] == [fpk[0][2], fpk[2][2]]
    assert [m["PT"] for m in members_of(out[t[2][0]: t[2][0] + t[2][1]])] == [pj.PT_REQUEST]
    e.close()
    f.close()


@pytest.mark.parametrize("wrap", [MAX_MEMBER + WRAP_OVERHEAD + 1, MAX_MEMBER + WRAP_OVERHEAD + 600])
def test_small_wrappers_cut_often_with_forwards(lib, wrap):
    rng = np.random.default_rng(wrap)
    world, fwd = random_case(rng, 2, n_groups=12, n_req=400, batching=0)
    e, named = world_emu(lib, world)
    rep, dec = json_replies(rng, world, 200, 2), json_decisions(rng, world, 200)
    out, refs, _ = check(e, world, named, rep, dec, fwd, wrap=wrap)
    wrappers = [p for p in pkts_of(out, refs) if p.startswith(b'{"type":90,"PT":37')]
    assert len(wrappers) > 20 and max(len(w) for w in wrappers) <= wrap
    e.close()


def test_erange_writes_nothing_and_einval(lib):
    rng = np.random.default_rng(12)
    world, fwd = random_case(rng, 3, n_groups=20, n_req=120)
    e, named = world_emu(lib, world)
    rep, dec = json_replies(rng, world, 40, 3), json_decisions(rng, world, 40)
    _, _, _, eout, erefs, _ = expected_sweep(world, named, rep, dec, fwd)
    for caps in ([0, 0], [len(eout) - 1, len(erefs)], [len(eout), len(erefs) - 1]):
        rc, _, _, _, out, refs, sz = sweep(e, rep, dec, fwd, sizes=caps)
        assert rc == abi.GPX_ERANGE and list(sz) == [len(eout), len(erefs)]
        assert (out == 0xCD).all() and (refs["len"] == 0).all()
    rc, _, _, _, out, _, _ = sweep(e, rep, dec, fwd, sizes=[len(eout), len(erefs)])
    assert rc == 0 and bytes(out[: len(eout)]) == eout
    assert sweep(e, rep, dec, fwd, wrap=MAX_MEMBER + WRAP_OVERHEAD)[0] == abi.GPX_EINVAL
    assert sweep(e, rep, dec, fwd, wrap=(4 << 20) + 1)[0] == abi.GPX_EINVAL
    # an oversized commit member fails the sweep, forwards or not
    gid = next(g for g, (_, _, m) in world.groups.items() if any(world.lane_of(x) is None for x in m))
    big = np.zeros(6000, abi.decision_dtype)
    big["gid"], big["slot"], big["bnum"], big["bcoord"] = gid, np.arange(6000) - (1 << 31), 1, world.groups[gid][2][0]
    big["flags"] = abi.F_DECISION
    rc = sweep(e, None, big, fwd, sizes=[1 << 24, 1 << 16])
    assert rc[0] == abi.GPX_EINVAL and (rc[4] == 0xCD).all()
    e.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_sweep_decodes_to_the_byte_forwards_requests(lib, fwd_lib, seed):
    """the sender's lanes (100, 101, 102); the receiver serves the other nodes: the JSON members through
    gpx_wire_decode_json_device and gpx_wire_decode_json_requests_device, and the lone packets through
    gpx_wire_decode_requests_device, give the requests the forwards encoder's packets decode to (client aside)"""
    rng = np.random.default_rng(seed)
    world, fwd = random_case(rng, 3, n_groups=200, n_req=400, **[dict(), dict(max_batch_size=2)][seed - 1])
    tx, named = world_emu(lib, world)
    rep, dec = json_replies(rng, world, 60, 3), json_decisions(rng, world, 60)
    rep["who"] &= ~np.uint32(abi.F_NACK << 16)
    _, _, _, rq, out, refs, _ = sweep(tx, rep, dec, fwd)
    rows, reqs, meta, status, payload, down = fwd
    fx = Emu(fwd_lib, world)
    _, fpk = encode_forwards(fx, rows, reqs, meta, status, payload, down)
    rx = Emu(fwd_lib, World(world.groups, [98, 99, 103, 104]))
    pk = [(out[int(r["off"]): int(r["off"]) + int(r["len"])], int(r["node"])) for r in refs]
    arena, prefs, nb = arena_of(pk)
    pst, mem = decode_members(rx, arena, prefs, nb)
    rc, _, jreqs, jmeta, jpay, _ = decode_json_requests(rx, arena, prefs, nb, mem)
    assert rc == 0
    lone = [p for p in pk if not p[0].startswith(b"{")]
    _, lreqs, lmeta, lpay = decode_requests(rx, lone) if lone else (None, jreqs[:0], jmeta[:0], jpay[:0])
    _, breqs, bmeta, bpay = decode_requests(rx, [(b, n) for _, n, b in fpk])

    def multiset(rq_, mt, pay):
        mt = mt.copy()  # NFWDS is written only when positive (toJSONSmartImpl): a count below 1 reads back as 0
        mt["forward_count"] = np.maximum(mt["forward_count"], 0)
        return sorted((r["gid"], r["flags"], r["req_id"], r["entry_node"], m.tobytes(),
                       bytes(pay[int(r["payload_off"]): int(r["payload_off"]) + int(r["payload_len"])]))
                      for r, m in zip(rq_, mt))
    assert sorted(multiset(jreqs, jmeta, jpay) + multiset(lreqs, lmeta, lpay)) == multiset(breqs, bmeta, bpay)
    assert len(jreqs) > 20 and len(lreqs) > 20
    assert len(breqs) == int((rq == abi.WE_SENT).sum())  # every request sent arrives once
    tx.close()
    fx.close()
    rx.close()


def test_wire_json_sweep_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_wire_json_sweep.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
