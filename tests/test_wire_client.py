"""CPU: gpx_wire_decode_client_requests_device's sequence and k_json_client (gigapaxos_b200/csrc/gpx_wire_fwd.cuh)
compiled for the host (tests/emu/wire_client_emu.cpp), against the model of tests/wire_client_cases.py.

* Random client traffic -- org.json and json-smart objects, QV bytes raw, escaped or \\u00XX, receiver stamps in the
  org.json, json-smart and "host/" forms, connections with unknown ports, batched requests, unknown names, stale
  versions, digests, responses, non-local nodes, and byteified REQUESTs, wrappers and other JSON among them -- decodes
  to the model's statuses, requests, meta and payload byte for byte, with and without peers.
* The same requests with the resolved "CA" / "LA" written out decode to the same outputs through
  gpx_wire_decode_json_requests_device's sequence.
* A corpus with one rule per case; GPX_ERANGE.
* Every output the same in ascending, descending and shuffled thread orders; the module once more in child runs under
  desc and two shuffles, and under AddressSanitizer + UBSan."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, abi, emu_library, ptr
from test_wire_dev import Emu
from test_wire_forward import arena_of, decode_json_requests
from wire_client_cases import corpus, expected, peer_rows, random_client_packets, random_resolvable
from wire_coord_cases import NOW_MS
from wire_dev_cases import random_world


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emu_library(tmp_path_factory, "wire_client_emu")


def decode_clients(e: Emu, arena, refs, nb, peers, sizes=None, block=64):
    """(rc, status, reqs, meta, payload, sizes); peers: wire_peer_dtype rows or None; sizes = the capacities (None:
    the sizes first)"""
    n = len(refs)
    status = np.full(max(n, 1), -9, np.int32)
    cap = np.array(sizes if sizes is not None else [0, 0], np.uint64)
    go = lambda cap, rq, mt, pay: e.lib.emu_wire_decode_client_requests(
        e.h, C.c_uint32(n), ptr(arena), C.c_uint64(nb), ptr(refs), None if peers is None else ptr(peers),
        C.c_int64(NOW_MS), ptr(status), ptr(rq), ptr(mt), ptr(pay), ptr(cap), C.c_uint32(block))
    if sizes is None:
        z = np.zeros(16, np.uint8)
        assert go(cap, z, z, z) in (0, abi.GPX_ERANGE)
    reqs = np.zeros(max(int(cap[0]), 1), abi.request_dtype)
    meta = np.zeros(max(int(cap[0]), 1), abi.req_meta_dtype)
    pay = np.zeros(max(int(cap[1]), 16), np.uint8)
    rc = go(cap, reqs, meta, pay)
    return rc, status[:n], reqs[: int(cap[0])], meta[: int(cap[0])], pay[: int(cap[1])], cap


def whole_members(refs):
    """a member table whose members are the whole packets, as gpx_wire_decode_json_device lists a bare packet"""
    mem = np.zeros(max(len(refs), 1), abi.wire_member_dtype)
    mem["pkt"][: len(refs)] = np.arange(len(refs))
    mem["off"][: len(refs)], mem["len"][: len(refs)] = refs["off"], refs["len"]
    mem["status"] = abi.WS_UNHANDLED
    return mem[: len(refs)]


def assert_as_model(got, want):
    rc, st, reqs, meta, pay, _ = got
    est, ereqs, emeta, epay = want
    assert rc == 0
    assert st.tolist() == est.tolist()
    assert reqs.tobytes() == ereqs.tobytes() and meta.tobytes() == emeta.tobytes()
    assert pay.tobytes() == epay.tobytes()


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("block", [1, 64])
def test_client_packets_decode_as_the_model(emu, seed, block):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 40)
    e = Emu(emu, world)
    pkts, peers = random_client_packets(rng, world, 400)
    arena, refs, nb = arena_of(pkts)
    for given in (True, False):
        got = decode_clients(e, arena, refs, nb, peer_rows(peers) if given else None, block=block)
        want = expected(world, pkts, peers if given else None)
        assert_as_model(got, want)
        seen = set(want[0].tolist())
        assert {abi.WS_OK, abi.WS_UNKNOWN_NAME, abi.WS_VERSION, abi.WS_UNHANDLED, abi.WS_NOT_LOCAL} <= seen
        assert len(got[2]) > 400
    # with peers, the requests without an address took their connection's; without, they stay all zeros
    m_with = decode_clients(e, arena, refs, nb, peer_rows(peers))[3]
    assert (m_with["client_port"] != 0).mean() > 0.3
    e.close()


@pytest.mark.parametrize("seed", [4, 5])
def test_outputs_are_the_json_requests_decoders_with_the_addresses_written_out(emu, seed):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 30)
    e = Emu(emu, world)
    pkts, peers, inserted = random_resolvable(rng, world, 300)
    arena, refs, nb = arena_of(pkts)
    got = decode_clients(e, arena, refs, nb, peer_rows(peers))
    ia, ir, inb = arena_of(inserted)
    ref = decode_json_requests(e, ia, ir, inb, whole_members(ir))
    assert got[0] == ref[0] == 0
    assert got[1].tolist() == ref[1].tolist() and (got[1] == abi.WS_OK).sum() > 150
    for a, b in zip(got[2:5], ref[2:5]):
        assert a.tobytes() == b.tobytes()
    assert_as_model(got, expected(world, pkts, peers))
    e.close()


def test_one_rule_per_case(emu):
    rng = np.random.default_rng(9)
    world = random_world(rng, 20)
    e = Emu(emu, world)
    cases = corpus(world)
    for with_peers in (True, False):
        sel = [c for c in cases if (c[2] is not None) == with_peers]
        arena, refs, nb = arena_of([(b, node) for b, node, _, _, _ in sel])
        peers = [c[2] for c in sel]
        rc, st, reqs, meta, pay, _ = decode_clients(e, arena, refs, nb, peer_rows(peers) if with_peers else None)
        assert rc == 0 and st.tolist() == [c[3] for c in sel]
        assert_as_model((rc, st, reqs, meta, pay, None),
                        expected(world, [(b, node) for b, node, _, _, _ in sel], peers if with_peers else None))
        # the outer request's addresses (the first record of each OK packet: the client column is the packet index)
        addr = lambda ip, port: (".".join(str(int(x)) for x in ip), int(port)) if int(port) else None
        for k, c in enumerate(sel):
            if c[4] is None:
                continue
            q = int(np.flatnonzero(reqs["client"] == k)[0])
            assert (addr(meta[q]["client_ip"], meta[q]["client_port"]), addr(meta[q]["listen_ip"],
                                                                             meta[q]["listen_port"])) == c[4], k
            # its BATCH entries take no connection address
            for p in np.flatnonzero(reqs["client"] == k)[1:]:
                assert addr(meta[p]["client_ip"], meta[p]["client_port"]) in (None, ("7.7.7.7", 7), ("6.6.6.6", 6))
                assert int(meta[p]["listen_port"]) == 0
    batched = [c for c in cases if b'"BATCH":[{' in c[0] and c[3] == abi.WS_OK]
    assert batched
    e.close()


def test_capacity_and_arguments(emu):
    rng = np.random.default_rng(11)
    world = random_world(rng, 20)
    e = Emu(emu, world)
    pkts, peers = random_client_packets(rng, world, 120, mixed=False)
    arena, refs, nb = arena_of(pkts)
    pr = peer_rows(peers)
    rc, _, _, _, _, need = decode_clients(e, arena, refs, nb, pr)
    assert rc == 0 and need[0] > 0
    for caps in ([int(need[0]) - 1, int(need[1])], [int(need[0]), int(need[1]) - 1]):
        rc, _, reqs, meta, pay, got = decode_clients(e, arena, refs, nb, pr, sizes=caps)
        assert rc == abi.GPX_ERANGE and got.tolist() == need.tolist()
        assert not reqs.tobytes().strip(b"\0") and not meta.tobytes().strip(b"\0") and not pay.tobytes().strip(b"\0")
    # a ref past the arena is malformed; no packets is nothing
    bad = refs.copy()
    bad["off"][0] = nb - 2
    rc, st, _, _, _, _ = decode_clients(e, arena, bad, nb, pr)
    assert rc == 0 and st[0] == abi.WS_MALFORMED
    rc, st, reqs, _, _, got = decode_clients(e, arena, refs[:0], nb, pr)
    assert rc == 0 and len(st) == 0 and got.tolist() == [0, 0]
    e.close()


# ---- thread orders and sanitizers -------------------------------------------------------------------------------------
def test_same_outputs_in_every_thread_order(emu):
    from test_emu_orders import contended_world, same_in_every_order
    rng = np.random.default_rng(12)
    world = contended_world(rng, 120)
    pkts, peers = random_client_packets(rng, world, 400)
    arena, refs, nb = arena_of(pkts)
    pr = peer_rows(peers)
    unnamed = list(world.groups)[::6]

    def run():
        e = Emu(emu, world)
        e.remove(unnamed)
        out = [decode_clients(e, arena, refs, nb, pr, block=7), decode_clients(e, arena, refs, nb, None, block=7)]
        e.close()
        return out
    out = same_in_every_order(emu, run)
    assert out[0][2][1][0] > 300


def _child(env_extra):
    env = dict(os.environ, **env_extra)
    return subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                           os.path.join(ROOT, "tests", "test_wire_client.py"), "-k",
                           "not asan and not thread_order and not in_order"],
                          capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)


@pytest.mark.parametrize("spec", ["desc", "shuffle:1", "shuffle:20261018"])
def test_module_passes_in_order(spec):
    if os.environ.get("GPX_EMU_ORDER") or os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already a child run")
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no CUDA headers")
    r = _child({"GPX_EMU_ORDER": spec})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and " failed" not in r.stdout


def test_client_kernel_is_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE") or os.environ.get("GPX_EMU_ORDER"):
        pytest.skip("already a child run")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    r = _child({"GPX_EMU_SANITIZE": "1", "LD_PRELOAD": asan, "ASAN_OPTIONS": "detect_leaks=0:abort_on_error=0"})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
