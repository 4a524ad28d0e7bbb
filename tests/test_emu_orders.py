"""CPU: the emulated kernels (tests/emu) in other thread orders than ascending.  On the device the threads and blocks of a
launch run in no fixed order; emu_launch runs them in the order GPX_EMU_ORDER names (asc, desc, shuffle:<seed>), so a
kernel whose output follows that order -- a thread reading what another thread of the launch writes, two threads writing
one place, an output laid out in the order of an atomicAdd or atomicCAS -- gives a different answer here too.

* the probe kernels (tests/emu/order_probe_emu.cpp) show that the order reaches a launch, in-process and through the
  environment of the child runs;
* the emulated-kernel modules run once more in child pytest runs under desc and two shuffle seeds;
* every emulated entry point runs the same call under asc, desc and shuffles in one process, on inputs where many
  threads contend for one atomic target, and every output byte the ABI defines, and the state the call leaves, must
  be the same.

Out of reach: interleaving inside a thread (each thread still runs to completion before the next starts), the kernels
tests/emu cannot run (k_round, k_round_g, the phase kernels) and the CUB side of the CUDA executor."""
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from helpers import ROOT, abi, emu_libraries, ptr

SHUFFLES = ("shuffle:1", "shuffle:20261018")
ORDERS = ("desc",) + SHUFFLES
MODULES = ("test_phase1b.py", "test_pause_batch.py", "test_log_find.py",
           "test_wire_dev.py", "test_wire_device.py", "test_wire_coord.py", "test_wire_forward.py",
           "test_wire_json.py", "test_wire_json_out.py", "test_wire_json_sweep.py",
           "test_rc_cpu.py", "test_journal_frames.py", "test_journal_gc.py")


class order:
    """`with order(lib, "shuffle:7"):` runs lib's launches in that order, then goes back to GPX_EMU_ORDER"""

    def __init__(self, lib, spec):
        self.lib, self.spec = lib, spec

    def __enter__(self):
        assert self.lib.emu_set_order(self.spec.encode()) == 0, self.spec

    def __exit__(self, *exc):
        self.lib.emu_set_order(None)


# --- the probe ------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    lib = emu_libraries(tmp_path_factory, "order_probe_emu")["order_probe_emu"]
    lib.emu_probe_chain.argtypes = lib.emu_probe_append.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    return lib


def probe_outputs(lib, n=200, block=7):
    chain, append = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    lib.emu_probe_chain(ptr(chain), n, block)
    lib.emu_probe_append(ptr(append), n, block)
    return chain, append


def test_the_probe_follows_the_order_set_in_process(probe):
    ident = np.arange(200, dtype=np.uint32)
    seen = []
    for spec in ("asc",) + ORDERS:
        with order(probe, spec):
            chain, append = probe_outputs(probe)
        assert sorted(append.tolist()) == ident.tolist(), spec  # every thread ran exactly once
        if spec == "asc":
            assert (chain == ident).all() and (append == ident).all()
        else:
            assert not (chain == ident).all() and not (append == ident).all(), spec
        seen.append(append.tobytes())
    assert len(set(seen)) == len(seen)  # desc and each seed are different orders
    if not os.environ.get("GPX_EMU_ORDER"):
        assert (probe_outputs(probe)[1] == ident).all()  # back to the environment's order
    for bad in ("", "up", "shuffle:", "shuffle:x", "shuffle:-1", "desc "):
        assert probe.emu_set_order(bad.encode()) == (0 if bad == "" else -1), bad
    probe.emu_set_order(None)


def test_the_probe_follows_the_environment(probe):
    """run in every child below: a mistake in passing GPX_EMU_ORDER through would let every order pass untested"""
    ident = np.arange(200, dtype=np.uint32)
    chain, append = probe_outputs(probe)
    assert sorted(append.tolist()) == ident.tolist()
    spec = os.environ.get("GPX_EMU_ORDER", "asc")
    if spec == "asc":
        assert (chain == ident).all() and (append == ident).all()
    else:
        assert not (chain == ident).all() and not (append == ident).all(), spec
        if spec == "desc":
            assert (append == ident[::-1]).all()


def test_a_shuffle_replays_by_seed_and_test(probe):
    """the same seed gives the same orders in the same test phase; the launch count moves the order on"""
    with order(probe, "shuffle:5"):
        a, b = probe_outputs(probe)[1], probe_outputs(probe)[1]
    env = dict(os.environ, GPX_EMU_ORDER="shuffle:5", PYTEST_CURRENT_TEST="replay")
    code = ("import ctypes as C, numpy as np, sys; lib = C.CDLL(sys.argv[1]);"
            "o = [np.zeros(200, np.uint32) for _ in range(2)];"
            "[lib.emu_probe_append(C.c_void_p(x.ctypes.data), 200, 7) for x in o];"
            "print(o[0].tobytes().hex(), o[1].tobytes().hex())")
    runs = [subprocess.run([sys.executable, "-c", code, probe._name], env=env, capture_output=True, text=True,
                           check=True).stdout.split() for _ in range(2)]
    assert runs[0] == runs[1] and runs[0][0] != runs[0][1]
    assert not (a == b).all()


# --- the emulated-kernel modules in other orders --------------------------------------------------------------------

def child_command():
    return [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-m", "not gpu",
            *[os.path.join("tests", m) for m in MODULES],
            "tests/test_emu_orders.py::test_the_probe_follows_the_environment", "-k", "not asan and not sanitized"]


@pytest.fixture(scope="module")
def children(request):
    """one child pytest per order this session runs, all started at once: each is about two minutes of one core"""
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no CUDA headers")
    wanted = [it.callspec.params["spec"] for it in request.session.items
              if it.module is request.module and it.originalname == "test_emulated_kernels_pass_in_order"]
    runs = {}
    for spec in dict.fromkeys(wanted):
        env = dict(os.environ, GPX_EMU_ORDER=spec)
        env.pop("GPX_EMU_SANITIZE", None)
        runs[spec] = (subprocess.Popen(child_command(), cwd=ROOT, env=env, stdout=subprocess.PIPE,
                                       stderr=subprocess.STDOUT, text=True), time.time())
    yield runs
    for p, _ in runs.values():
        if p.poll() is None:
            p.kill()
            p.wait()


@pytest.mark.parametrize("spec", ORDERS)
def test_emulated_kernels_pass_in_order(children, spec):
    p, t0 = children[spec]
    out, _ = p.communicate(timeout=1800)
    wall = time.time() - t0
    repro = f"GPX_EMU_ORDER={spec} " + " ".join(child_command()[1:])
    assert p.returncode == 0, f"GPX_EMU_ORDER={spec}: child failed after {wall:.0f} s; replay with\n  {repro}\n{out[-6000:]}"
    assert " passed" in out and " failed" not in out, out[-3000:]
    print(f"GPX_EMU_ORDER={spec}: {out.strip().splitlines()[-1]} ({wall:.0f} s)")


# --- every emulated entry point: the same call in every order, in one process ---------------------------------------
# A test holds an output against what its model predicts, and a lenient model could hide an order effect; here each
# entry point's outputs and the state it leaves are held against its own asc run, byte for byte, on inputs where many
# threads contend for one atomic target.

SAME = ("asc", "desc", "shuffle:1", "shuffle:2", "shuffle:3", "shuffle:20261018")
SOURCES = ("wire_json_sweep_emu", "wire_fwd_emu", "rc_emu", "journal_emu", "journal_gc_emu", "p1b_emu", "pause_emu",
           "logfind_emu")
U32, U64, P = C.c_uint32, C.c_uint64, C.c_void_p
SIGNATURES = {
    "emu_wire_new": ([U32, U32, P], P),
    "emu_journal_new": ([U32, U32], P),
    "emu_journal_free": ([P], None),
    "emu_journal_names": ([P, U32, P, P, P], None),
    "emu_journal_names_remove": ([P, U32, P], None),
    "emu_log_frame": ([P, P, U64, U64, P, P, U32, P, P, P, U32], C.c_int),
    "emu_jgc_new": ([U32], P),
    "emu_jgc_free": ([P], None),
    "emu_jgc_names": ([P, U32, P, P, P, P], None),
    "emu_jgc_compact": ([P, P, U64, P, U32, P, U32, P, U32, U32, P, P, P, P, U32], C.c_int),
    "emu_jgc_index": ([P, U64, U32, P, U32, P, P], C.c_int),
    "emu_log_find": ([P, U64, U64, U64, U32, U32, P, P, U32, U32], C.c_int),
    "emu_log_gather": ([P, U64, U64, U32, U32, P, P, U64, U32], C.c_int),
}


@pytest.fixture(scope="module")
def emus(tmp_path_factory):
    """every emulated entry point: source -> library"""
    libs = emu_libraries(tmp_path_factory, *SOURCES)
    for lib in libs.values():
        for f, (args, res) in SIGNATURES.items():
            if hasattr(lib, f):
                getattr(lib, f).argtypes, getattr(lib, f).restype = args, res
    return libs


def canon(x):
    if isinstance(x, np.ndarray):
        return (x.dtype.str, x.shape, x.tobytes())
    if isinstance(x, (list, tuple)):
        return tuple(canon(y) for y in x)
    return repr(x) if hasattr(x, "__dataclass_fields__") else x


def n_rows(c):
    """the length of an array that canon() turned into (dtype, shape, bytes)"""
    return c[1][0]


def same_in_every_order(lib, run):
    """run() -- which sets up fresh state, makes its calls and returns what they wrote -- under asc, desc and four
    shuffles: every output of every order is asc's, byte for byte"""
    got = {}
    for spec in SAME:
        with order(lib, spec):
            got[spec] = canon(run())
    want = got["asc"]
    for spec in SAME[1:]:
        assert len(got[spec]) == len(want)
        for k, (a, b) in enumerate(zip(want, got[spec])):
            assert a == b, f"GPX_EMU_ORDER={spec}: output {k} is not what asc wrote"
    return want


def hash_alike(k):
    """names that share one String.hashCode in blocks of 64 ("Aa" and "BB" hash alike), the blocks on neighbouring
    hashes: every insert of a block probes one run of table cells"""
    return "".join("Aa" if (k >> b) & 1 else "BB" for b in range(6)) + chr(0x30 + k // 64)


def contended_world(rng, n_groups, lanes=(100, 101, 102)):
    """wire_dev_cases.random_world under hash_alike names, most groups on one of two member sets (the JSON encoder's
    recipient sets then have many members each)"""
    from wire_dev_cases import World, random_world
    sets = ([100, 101, 103], [100, 102, 103, 104])
    base = random_world(rng, n_groups, lanes)
    return World({g: (hash_alike(g), v, m if g % 5 == 0 else sets[g % 2]) for g, (_, v, m) in base.groups.items()},
                 lanes)


def test_name_table_calls_in_every_order(emus):
    """emu_wire_names (find, remove, store, insert), emu_wire_names_remove and emu_wire_names_rehash.  gpx.h gives the
    name state as "an open-addressing table of 8-byte cells (at least 2 per gid)" and says nothing of which cell holds a
    name, so the table is compared through lookups: which gid each name finds, and each packet's status"""
    from test_wire_dev import Emu
    from gigapaxos_b200 import wire
    lib = emus["wire_json_sweep_emu"]
    world = contended_world(np.random.default_rng(1), 300)
    gids = list(world.groups)
    commits = [wire.encode_batched_commit(world.groups[g][0], world.groups[g][1], 1, world.groups[g][2][0], 0, [1],
                                          world.groups[g][2]) for g in gids]

    def run():
        e = Emu(lib, world)
        out = [e.set_names(gids)]  # every name found at its own gid
        e.remove(gids[::3])
        out.append(e.decode(commits, 7)[0])
        out.append(e.set_names(gids[::3]))  # not found: removed
        for _ in range(2):
            e.remove(gids[1::4])
            e.set_names(gids[1::4])
        out.append(e.decode(commits, 7)[0])
        lib.emu_wire_names_rehash(e.h)
        out += [e.decode(commits, 7)[0], e.set_names(gids)]
        e.close()
        return out
    out = same_in_every_order(lib, run)
    assert out[0] == canon(np.array(gids, np.uint32)) and out[-1] == out[0]


def test_byte_codec_calls_in_every_order(emus):
    """emu_wire_decode, emu_wire_decode_requests and emu_wire_encode (replies, decisions, ACCEPTs with their requests)"""
    from test_wire_coord import decode_requests, encode_accepts
    from test_wire_dev import Emu
    from wire_coord_cases import random_accepts, random_request_packets
    from wire_dev_cases import random_decisions, random_packets, random_replies
    lib = emus["wire_json_sweep_emu"]
    rng = np.random.default_rng(2)
    world = contended_world(rng, 150)
    pkts, _ = random_packets(rng, world, 400)
    rpkts = random_request_packets(rng, world, 400)
    rep = random_replies(rng, world, 300, 3)
    dec = random_decisions(rng, world, 400)
    accs = random_accepts(rng, world, 60)
    unnamed = list(world.groups)[::7]

    def run():
        e = Emu(lib, world)
        e.remove(unnamed)
        out = [e.decode(pkts, 7), decode_requests(e, rpkts, 7), e.encode(rep, 1, 7), e.encode(dec, 0, 7),
               encode_accepts(e, *accs, block=7)]
        e.close()
        return out
    out = same_in_every_order(lib, run)
    assert len(out[2][1]) > 10 and len(out[3][1]) > 10 and len(out[4][1]) > 10


def test_json_calls_in_every_order(emus):
    """emu_wire_decode_json, emu_wire_encode_json and emu_wire_encode_json_sweep; the encoders' first member of each
    (lane, recipient set) is an atomicMin over many members"""
    from test_wire_dev import Emu
    from test_wire_json import decode_json
    from test_wire_json_out import encode_json
    from test_wire_json_sweep import edge_values, sweep
    from wire_fwd_cases import forward_case
    from wire_json_cases import as_json, group_into_packets, random_logical
    from wire_json_out_cases import json_decisions, json_replies
    lib = emus["wire_json_sweep_emu"]
    rng = np.random.default_rng(3)
    world = contended_world(rng, 120)
    js, _ = group_into_packets(rng, [as_json(k, f, rng) for k, f in random_logical(rng, world, 200)])
    rep = json_replies(rng, world, 200, 3)
    dec = json_decisions(rng, world, 300)
    fwd = forward_case(rng, world, 300, max_batch_size=3)
    edge_values(rng, fwd[1], fwd[2])
    unnamed = list(world.groups)[::9]

    def run():
        e = Emu(lib, world)
        e.remove(unnamed)
        out = [decode_json(e, js, block=7), encode_json(e, rep, dec, block=7), encode_json(e, rep, dec, wrap=600, block=7),
               sweep(e, rep, dec, fwd, block=7), sweep(e, rep, dec, fwd, wrap=600, block=7)]
        e.close()
        return out
    out = same_in_every_order(lib, run)
    assert n_rows(out[0][1]) > 100 and n_rows(out[1][4]) > 10 and n_rows(out[3][5]) > 10


def test_forward_calls_in_every_order(emus):
    """emu_wire_encode_forwards and emu_wire_decode_json_requests"""
    from test_wire_dev import Emu
    from test_wire_forward import arena_of, decode_json_requests, decode_members, encode_forwards
    from wire_coord_cases import random_request_packets
    from wire_fwd_cases import forward_case, json_wrappers
    lib = emus["wire_fwd_emu"]
    rng = np.random.default_rng(4)
    world = contended_world(rng, 120)
    rows, reqs, meta, status, payload, down = forward_case(rng, world, 500, max_batch_size=2)
    wraps, _ = json_wrappers(world, random_request_packets(rng, world, 300), rng)
    arena, refs, nb = arena_of(wraps)
    unnamed = list(world.groups)[::6]

    def run():
        e = Emu(lib, world)
        e.remove(unnamed)
        out = [encode_forwards(e, rows, reqs, meta, status, payload, down, block=7),
               encode_forwards(e, rows, reqs, meta, status, payload, (), block=7)]
        mem = decode_members(e, arena, refs, nb)
        out += [mem, decode_json_requests(e, arena, refs, nb, mem[1], block=7)]
        e.close()
        return out
    out = same_in_every_order(lib, run)
    assert len(out[0][1]) > 10 and n_rows(out[3][2]) > 300


def test_response_cache_calls_in_every_order(emus):
    """emu_rc_gen_bump, emu_rc_put and emu_rc_match: puts of thousands of keys drawn from a pool of eight, so one batch
    holds each key many times, into a table of 16 buckets"""
    from rc_cases import random_keys, random_requests
    from test_rc_cpu import EmuCache
    lib = emus["rc_emu"]
    rng = np.random.default_rng(5)
    G = 64
    pool = [(int(rng.integers(G)), int(rng.integers(1 << 40)), ((10, 0, 0, i % 4), 1000 + i % 3)) for i in range(8)]
    ops = [(random_keys(rng, 3000, G, pool), random_requests(rng, 1000, G, pool)) for _ in range(3)]

    def run():
        e = EmuCache(lib, 16, 1000, G, True, 7)
        e.name(list(range(0, G, 2)))
        e.name(list(range(0, G, 3)))
        out = [e.gen.copy()]
        for r, (keys, (reqs, meta)) in enumerate(ops):
            out += [e.put(keys, 10 * r), e.cells.copy(), e.match(reqs, meta, 10 * r + 5)]
        return out
    out = same_in_every_order(lib, run)
    assert sum(int((canon_hits >= 0).sum()) for canon_hits in (np.frombuffer(h[0][2], np.int32) for h in out[3::3])) > 100


def colliding_names(G):
    return {g: hash_alike(g).encode() + (b"\\" if g % 3 == 0 else b"") for g in range(G)}


def test_journal_frame_calls_in_every_order(oracle_lib, emus):
    """emu_journal_names, emu_journal_names_remove and emu_log_frame on the oracle engine's rings, names colliding in
    the table"""
    from test_journal_frames import Emu, make_meta, oracle_ring, requests_of
    from test_log_find import logged_engine
    lib = emus["journal_emu"]
    G = 40
    eng, _ = logged_engine(oracle_lib, G, seed=6)
    rng = np.random.default_rng(6)
    names = colliding_names(G)
    versions = {g: int(rng.integers(0, 3)) for g in range(G)}
    rings = [oracle_ring(eng, lane) for lane in range(3)]
    metas = [make_meta(requests_of(ring, cap, head, 0), rng) for ring, cap, head in rings]
    eng.close()
    gone = np.arange(0, G, 5, dtype=np.uint32)

    def run():
        e = Emu(lib, G, names, versions)
        out = [e.frame(ring, cap, head, 0, meta, block=7) for (ring, cap, head), meta in zip(rings, metas)]
        lib.emu_journal_names_remove(e.h, len(gone), ptr(gone))
        out += [e.frame(ring, cap, head, 0, meta[::2], block=7) for (ring, cap, head), meta in zip(rings, metas)]
        e.close()
        return out
    out = same_in_every_order(lib, run)
    assert all(o[0] == 0 for o in out[:3]) and all(o[0] == abi.GPX_ENOENT for o in out[3:])


def test_journal_gc_calls_in_every_order(oracle_lib, emus, tmp_path):
    """emu_jgc_names and emu_jgc_compact on the oracle engine's journals (a view change's PREPAREs: many frames of one
    group in the PREPARE rule's gid sort).  emu_jgc_index is a host walk and launches nothing."""
    from test_journal_frames import log_drainer, make_meta, oracle_ring, requests_of
    from test_journal_gc import Gc, gc_slots_for, roll
    from test_log_find import logged_engine
    lib = emus["journal_gc_emu"]
    G = 40
    eng, _ = logged_engine(oracle_lib, G, seed=7)
    rng = np.random.default_rng(7)
    names = colliding_names(G)
    versions = {g: int(rng.integers(0, 3)) for g in range(G)}
    live = {g: g % 7 != 3 for g in range(G)}
    probe_gc = Gc(lib, G, names, versions, live)
    cases = []
    for lane in range(3):
        ring, cap, head = oracle_ring(eng, lane)
        data, _ = log_drainer(ring, cap, head, 0, names, versions, make_meta(requests_of(ring, cap, head, 0), rng))
        blobs = roll(data, rng, 5)
        cases.append((blobs, gc_slots_for(blobs, probe_gc, rng)))
    probe_gc.close()
    eng.close()

    def run():
        g = Gc(lib, G, names, versions, live)
        out = [g.compact(blobs, gc, last_readonly=ro, block=7) for blobs, gc in cases for ro in (True, False)]
        g.close()
        return out
    out = same_in_every_order(lib, run)
    assert all(o[0] == 0 for o in out)


def test_prepare_tally_in_every_order(oracle_lib, emus):
    """emu_prepare_tally: its outputs and the rows, windows and nodeSlotNumbers it leaves"""
    from p1b_cases import NODES5, dump_all, make_engine, preconditions, random_elections
    from test_phase1b import _state_arrays
    lib = emus["p1b_emu"]
    R, G, W = 5, 160, 8
    rng = np.random.default_rng(8)
    eng = make_engine(oracle_lib, R, G, None)
    preconditions(eng, R, G, rng)
    els, reps = random_elections(R, G, rng, True, None)
    rows = dump_all(eng, R, G)
    state = _state_arrays(rows, R, G, W, R, rng)
    live = (rows[0]["state"] != abi.ST_FREE).astype(np.uint8)
    members = np.array(NODES5[:R], np.int32)

    def run():
        aux, crow, nsl, pwin = (a.copy() for a in state)
        got = np.zeros(len(els), abi.election_out_dtype)
        got.view(np.uint8)[:] = 0xAB
        assert lib.emu_prepare_tally(G, R, W, R, R, ptr(members), ptr(members), ptr(live), ptr(crow), ptr(aux), ptr(nsl),
                                     ptr(pwin), len(els), ptr(els), len(reps), ptr(reps), ptr(got), 7) == 1
        return [got, aux, crow, nsl, pwin]
    out = same_in_every_order(lib, run)
    verdicts = np.frombuffer(out[0][2], abi.election_out_dtype)["verdict"]
    assert (verdicts == abi.EL_MAJORITY).any()


def test_pause_select_and_missing_in_every_order(oracle_lib, emus):
    """emu_pause_groups (verdicts, rows, the state it leaves), emu_missing_decisions, emu_clear_group_flags, and
    emu_select_groups, whose kernel appends each match with one atomicAdd and whose gids the host sorts afterwards.
    With too small a buffer ("which `cap` of them were returned is unspecified", gpx.h) only their count and that they
    match are compared"""
    from test_pause_batch import NODES, busy_engine, pause_state
    lib = emus["pause_emu"]
    R, G, W = 3, 120, 8
    eng = busy_engine(oracle_lib, G, 9, 1, R)
    rng = np.random.default_rng(9)
    state = pause_state(eng, R, G, W, 0, rng)
    eng.close()
    gids = rng.permutation(G + 2).astype(np.uint32)
    nodes = np.array(NODES, np.int32)
    sweeps = [(lane, m, v) for lane in range(R) for m, v in ((abi.GF_NOT_CAUGHT_UP, 0), (0, 0),
                                                                (abi.GF_NOT_CAUGHT_UP, abi.GF_NOT_CAUGHT_UP))]

    def run():
        live, acc_row, acc_aux, acc_win, coord_row, node_slots = (a.copy() for a in state)
        out = []
        for lane, mask, value in sweeps:
            for cap in (G, 5):  # all matches fit, then too few
                found = np.zeros(cap, np.uint32)
                n = np.zeros(1, np.uint32)
                assert lib.emu_select_groups(G, R, W, R, R, ptr(nodes), ptr(nodes), ptr(live), 0, ptr(acc_row),
                                             ptr(acc_aux), ptr(acc_win), ptr(coord_row), lane, mask, value, ptr(found),
                                             cap, ptr(n), 7) == 1
                if int(n[0]) <= cap:
                    out.append(found[: int(n[0])])
                else:
                    assert np.isin(found, out[-1]).all()
                    out.append(n)
        for lane in range(R):
            miss = np.zeros(len(gids), abi.missing_dtype)
            miss.view(np.uint8)[:] = 0x5A
            assert lib.emu_missing_decisions(G, R, W, R, ptr(nodes), ptr(nodes), ptr(live), 1, ptr(acc_row),
                                             ptr(acc_aux), ptr(acc_win), ptr(coord_row), lane, len(gids), ptr(gids),
                                             400, 400, ptr(miss), 7) == 1
            out.append(miss)
        for lane in range(R):
            assert lib.emu_clear_group_flags(G, R, W, R, ptr(nodes), ptr(nodes), ptr(live), ptr(acc_aux), lane,
                                             len(gids) - lane, ptr(gids), abi.GF_NEEDS_SYNC << lane % 2, 7) == 0
        rows = np.zeros((len(gids), R), abi.row_dtype)
        ok = np.full(len(gids), 7, np.uint8)
        assert lib.emu_pause_groups(G, R, W, R, R, ptr(nodes), ptr(nodes), ptr(live), 0, ptr(acc_row), ptr(acc_aux),
                                    ptr(acc_win), ptr(coord_row), ptr(node_slots), len(gids), ptr(gids), ptr(rows),
                                    ptr(ok), 7) == 1
        return out + [rows, ok, acc_row, acc_aux, acc_win, coord_row, node_slots]
    out = same_in_every_order(lib, run)
    ok = np.frombuffer(out[-6][2], np.uint8)
    assert 0 < ok.sum() < len(gids)
    # the too-small buffers: each of them matched more than it holds, and what it holds are matches
    assert any(len(np.frombuffer(o[2], o[0])) == 1 for o in out[1: 2 * len(sweeps): 2])


def test_log_find_and_gather_in_every_order(oracle_lib, emus):
    """emu_log_find (k_log_scan's atomicMax cells: the same slots of every group accepted again and again, so each cell
    has many candidate images) and emu_log_gather"""
    from helpers import make_requests
    from test_log_find import logged_engine
    lib = emus["logfind_emu"]
    G = 40
    eng, _ = logged_engine(oracle_lib, G, seed=10)
    gids = np.arange(G, dtype=np.uint32)
    coord = np.array([[100, 101, 102].index(int(x)) for x in eng.dump_rows(gids, 0)["acc_bcoord"]])
    reqs, pay = make_requests(gids, payload_len=11, seed=10, round_no=0)
    reqs["flags"] = coord << 8
    reqs["entry_node"] = np.array([100, 101, 102])[coord]
    acc, blob, _ = eng.propose(reqs, pay)
    for reach in (0b111, 0b011, 0b110, 0b101, 0b111, 0b111):  # the same ACCEPTs, logged once per delivery
        a = acc.copy()
        a["dst_mask"] = reach
        eng.handle_accepts(a, blob)
    wants = np.zeros(G + 2, abi.log_want_dtype)
    wants["gid"], wants["min_slot"], wants["n_slots"] = np.arange(G + 2), 0, abi.GPX_LOG_SPAN
    rings = []
    for lane in range(3):
        buf = eng.log_read(lane)
        cap = 1 << int(np.ceil(np.log2(len(buf) + 64)))
        ring = np.zeros(cap, np.uint8)
        ring[: len(buf)] = buf
        hits = eng.log_find(lane, wants).reshape(-1)
        hits = hits[(hits["accept"]["flags"] & abi.F_VOID) == 0]
        r = np.zeros(len(hits), abi.log_range_dtype)
        r["pos"], r["len"] = hits["blob_pos"], hits["accept"]["payload_len"]
        padded = (r["len"].astype(np.uint64) + 15) // 16 * 16
        r["dst_off"] = np.concatenate([[0], np.cumsum(padded)[:-1]])
        rings.append((ring, cap, len(buf), r, int(padded.sum()) + 64))
    eng.close()

    def run():
        out = []
        for lane, (ring, cap, head, r, n_out) in enumerate(rings):
            for grid, block in ((3, 7), (5, 64)):
                hits = np.zeros((len(wants), abi.GPX_LOG_SPAN), abi.log_hit_dtype)
                hits.view(np.uint8)[:] = 0xCD
                assert lib.emu_log_find(ptr(ring), cap, head, 0, lane, len(wants), ptr(wants), ptr(hits), grid,
                                        block) == 1
                out.append(hits)
            gathered = np.full(n_out, 0xEE, np.uint8)
            assert lib.emu_log_gather(ptr(ring), cap, head, lane, len(r), ptr(r), ptr(gathered), n_out, 7) == 0
            out.append(gathered)
        return out
    out = same_in_every_order(lib, run)
    hits = np.frombuffer(out[0][2], abi.log_hit_dtype)
    assert ((hits["accept"]["flags"] & abi.F_VOID) == 0).sum() > G
