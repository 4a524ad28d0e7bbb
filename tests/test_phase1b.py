"""Phase 1b at the would-be coordinator (gpx_handle_prepare_replies; PISM.handlePrepareReply :1017-1068, PCS :264-587).

CPU: the oracle's entry point (a C++ restatement of the Java classes) against the host-language twin in
gigapaxos_b200/paxos_manager.py (tally_prepare_replies / combine_carryover + gpx_patch), a second, independently
structured restatement -- verdict, nodeSlotNumbers, plan and the rows both leave behind, over random elections."""
import numpy as np
import pytest

# GPX_EMU_SANITIZE=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) python -m pytest ... : the emulated kernels under
# AddressSanitizer + UBSan (every heap buffer numpy hands them gets red zones; so do their local arrays)
from gigapaxos_b200.paxos_manager import NoopPaxosApp, PaxosManager
from helpers import abi, emu_library, ptr
from p1b_cases import NODES5, assert_same_out, dump_all, make_engine, preconditions, random_elections


def twin_election(pm: PaxosManager, R: int, el, reps: np.ndarray):
    """the host-language twin on one election: -> election_out record (and the engine of `pm` patched as it patches)"""
    out = np.zeros(1, dtype=abi.election_out_dtype)[0]
    out["gid"], out["verdict"] = el["gid"], abi.EL_DROPPED
    out["node_slots"][:] = -1
    gid, lane = int(el["gid"]), int(el["lane"])
    eng = pm.engine
    if lane >= eng.n_lanes:
        return out
    row = eng.dump_rows(np.array([gid], dtype=np.uint32), lane)[0]
    if int(row["state"]) not in (abi.ST_ACTIVE_1, abi.ST_ACTIVE_2):
        return out
    # logical replies: a record and its GPX_F_MORE continuations (the twin takes the overflow as `logged`)
    logical, logged, first_rec = [], {}, []
    k, end = int(el["first_reply"]), int(el["first_reply"]) + int(el["n_replies"])
    while k < end:
        head = reps[k].copy()
        fl = abi.who_flags(int(head["who"]))
        extra = []
        first_rec.append(k)
        k += 1
        while (fl & abi.F_MORE) and not (fl & abi.F_VOID) and k < end:
            nxt = reps[k]
            extra += [(pv.copy(), k) for pv in nxt["accepted"][: int(nxt["n_accepted"])]]
            fl = abi.who_flags(int(nxt["who"]))
            k += 1
        logical.append(head)
        if extra:
            logged[len(logical) - 1] = extra
    my = (int(el["bnum"]), int(el["bcoord"]))
    # the twin reports the index of the logical reply; the engine the index of the RECORD: translate
    src_of = {}
    lg = {}
    for l, ex in logged.items():
        lg[l] = [pv for pv, _ in ex]
        for pv, rec in ex:
            src_of[(l, int(pv["slot"]))] = rec
    verdict, ns, carry = PaxosManager.tally_prepare_replies(logical, R, my, lg)
    out["node_slots"][:R] = ns
    out["verdict"] = {"waiting": abi.EL_WAITING, "majority": abi.EL_MAJORITY, "preempted": abi.EL_PREEMPTED,
                      "overflow": abi.EL_OVERFLOW}[verdict]
    if verdict != "majority":
        return out
    comb = PaxosManager.combine_carryover(carry, ns, int(el["slot"]))
    if comb is None:
        out["verdict"] = abi.EL_OVERFLOW
        return out
    plan, next_slot, flags = comb
    out["next_slot"], out["n_plan"], out["flags"] = next_slot, len(plan), flags
    for j, (sl, kind, pv, l) in enumerate(plan):
        c = out["plan"][j]
        c["slot"], c["kind"] = sl, kind
        if kind == abi.CO_PVALUE:
            c["pv"] = pv
            c["src_reply"] = src_of.get((l, int(pv["slot"])), first_rec[l])
    # ... and installs through gpx_patch exactly as PaxosManager._phase1b_host does
    res = pm._phase1b_host(gid, lane, R, my, int(el["slot"]), logical, lg)
    assert res is not None
    return out


@pytest.mark.parametrize("R,seed,wrap,lane_nodes", [(3, 1, False, None), (3, 2, True, None), (5, 3, False, None),
                                                    (5, 4, True, None), (1, 5, False, None), (4, 6, False, None),
                                                    (3, 7, False, [101]), (5, 8, True, [103, 100])])  # nodes of a spread placement
def test_oracle_phase1b_equals_the_host_twin(oracle_lib, R, seed, wrap, lane_nodes):
    G = 160
    rng = np.random.default_rng(seed)
    ea, eb = make_engine(oracle_lib, R, G, lane_nodes), make_engine(oracle_lib, R, G, lane_nodes)
    hosted = NODES5[:R] if lane_nodes is None else lane_nodes
    pm = PaxosManager(eb, [NoopPaxosApp() for _ in hosted], hosted)
    verdicts = set()
    for rnd in range(4):
        st = rng.bit_generator.state
        preconditions(ea, R, G, rng)
        rng.bit_generator.state = st
        preconditions(eb, R, G, rng)
        els, reps = random_elections(R, G, rng, wrap, lane_nodes)
        got = ea.handle_prepare_replies(els, reps)
        want = np.array([twin_election(pm, R, el, reps) for el in els], dtype=abi.election_out_dtype)
        assert_same_out(got, want)
        verdicts |= set(int(v) for v in got["verdict"])
        for ra, rb in zip(dump_all(ea, R, G), dump_all(eb, R, G)):
            for f in ra.dtype.names:
                assert np.array_equal(ra[f], rb[f]), f
    if R >= 3:
        assert verdicts == {abi.EL_WAITING, abi.EL_MAJORITY, abi.EL_PREEMPTED, abi.EL_DROPPED, abi.EL_OVERFLOW}


def test_phase1b_api_misuse(oracle_lib):
    eng = make_engine(oracle_lib, 3, 8)
    els = np.zeros(2, dtype=abi.election_dtype)
    els["gid"] = [1, 1]
    with pytest.raises(abi.GpxError):  # one election per group per call
        eng.handle_prepare_replies(els, np.zeros(0, dtype=abi.prepare_reply_dtype))
    els["gid"] = [1, 2]
    els["n_replies"] = [0, 3]
    with pytest.raises(abi.GpxError):  # replies out of range
        eng.handle_prepare_replies(els, np.zeros(2, dtype=abi.prepare_reply_dtype))
    assert len(eng.handle_prepare_replies(els[:0], np.zeros(0, dtype=abi.prepare_reply_dtype))) == 0


def test_elected_coordinator_proposes_the_plan(oracle_lib):
    """end to end on one group: two ACCEPTs reach a minority / a majority, the coordinator dies, the next node is elected
    by gpx_handle_prepare_replies and re-proposes the plan; the decided values are the carried-over ones, in slot order"""
    from test_paxos_manager import drive_view_change
    pm = drive_view_change(oracle_lib, p1b=True)
    assert pm.device_phase1b


# ---- the CUDA kernel's own source, run on the host ---------------------------------------------------------------------
# tests/emu/ compiles gigapaxos_b200/csrc/gpx_phase1b.cuh (k_prepare_tally as the GPU runs it: a scalar kernel over
# gpx_dev.cuh's structs and index helpers) with g++ and runs it thread by thread, driven by the engine's own host sequence
# (prepare_replies in gpx_state_seq.h: its checks, scratch layout, copies).  State goes in as the arrays DevState
# describes, taken from the oracle engine's rows before the call; outputs and the state the kernel leaves are held
# against the oracle's.  What this cannot see is the CUDA executor and the launch itself -- that is the GPU test's job
# (tests/test_zz_phase1b_gpu.py).
@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    return emu_library(tmp_path_factory, "p1b_emu")


def _state_arrays(rows, R, G, W, Rcap, rng):
    """DevState's arrays for phase 1b from dumped rows: acc_aux [L][G], coord_row [L][G] int4, node_slots [L][Rcap][G],
    prop_win [L][W][G] int4 (a nonzero pattern: only a resign / install may clear it)"""
    L = len(rows)
    aux = np.zeros((L, G), dtype=np.uint32)
    crow = np.zeros((L, G, 4), dtype=np.int32)
    nsl = np.full((L, Rcap, G), -7, dtype=np.int32)
    for l in range(L):
        r = rows[l]
        aux[l] = (r["state"].astype(np.uint32) & 0xFF) | (rng.integers(0, 1 << 16, size=G).astype(np.uint32) << 8)
        ex = r["coord_exists"] != 0
        crow[l, :, 0] = np.where(ex, r["coord_bnum"], 0)
        crow[l, :, 1] = np.where(ex, r["coord_bcoord"], 0)
        crow[l, :, 2] = np.where(ex, r["next_proposal_slot"], 0)
        crow[l, :, 3] = np.where(ex, 1 | np.where(r["coord_active"] != 0, 2, 0) | (rng.integers(0, 4, size=G) << 8), 0)
        nsl[l, :R, :] = r["node_slots"][:, :R].T
    pwin = rng.integers(1, 1 << 30, size=(L, W, G, 4)).astype(np.int32)
    return aux, crow, nsl, pwin


@pytest.mark.parametrize("R,seed,wrap,block,lane_nodes", [(3, 11, False, 64, None), (3, 12, True, 1, None), (5, 13, False, 64, None),
                                                          (5, 14, True, 7, None), (1, 15, False, 64, None), (4, 16, False, 33, None),
                                                          (3, 17, False, 64, [102]), (5, 18, True, 16, [101, 104])])
def test_kernel_source_on_the_host_equals_oracle(oracle_lib, emu_lib, R, seed, wrap, block, lane_nodes):
    G, W = 160, 8
    Rcap = R
    rng = np.random.default_rng(seed)
    eng = make_engine(oracle_lib, R, G, lane_nodes)
    L = eng.n_lanes
    for rnd in range(3):
        preconditions(eng, R, G, rng)
        els, reps = random_elections(R, G, rng, wrap, lane_nodes)
        rows = dump_all(eng, R, G)
        aux, crow, nsl, pwin = _state_arrays(rows, R, G, W, Rcap, rng)
        pwin0, crow0 = pwin.copy(), crow.copy()
        live = (rows[0]["state"] != abi.ST_FREE).astype(np.uint8)
        want = eng.handle_prepare_replies(els, reps)  # the oracle: outputs + its engine's new state
        got = np.zeros(len(els), dtype=abi.election_out_dtype)
        got.view(np.uint8)[:] = 0xAB  # the kernel must write every byte of its records
        members = np.array(NODES5[:R], dtype=np.int32)
        hosted = members if lane_nodes is None else np.array(lane_nodes, dtype=np.int32)
        launches = emu_lib.emu_prepare_tally(G, L, W, Rcap, R, ptr(members), ptr(hosted), ptr(live), ptr(crow), ptr(aux),
                                             ptr(nsl), ptr(pwin), len(els), ptr(els), len(reps), ptr(reps), ptr(got),
                                             block)
        assert launches == 1
        assert_same_out(got, want)
        if rnd == 0:  # the engine's refusals, before anything runs: replies beyond n_reply_recs, two elections of a group
            for k, (e2, n_reps, rc, error) in enumerate(((els, len(reps) - 1, abi.GPX_ERANGE, b"beyond n_reply_recs"),
                                                        (np.concatenate([els, els[:1]]), len(reps), abi.GPX_EINVAL,
                                                         b"more than one election"))):
                st = [a.copy() for a in (crow, aux, nsl, pwin)]
                if k == 0:
                    e2 = e2[np.argsort(e2["first_reply"] + e2["n_replies"])]  # the last reply is referred to
                bad = np.zeros(len(e2), dtype=abi.election_out_dtype)
                assert emu_lib.emu_prepare_tally(G, L, W, Rcap, R, ptr(members), ptr(hosted), ptr(live), ptr(st[0]),
                                                 ptr(st[1]), ptr(st[2]), ptr(st[3]), len(e2), ptr(e2), n_reps, ptr(reps),
                                                 ptr(bad), block) == rc
                assert error in emu_lib.emu_last_error() and not bad.view(np.uint8).any()
                assert all(np.array_equal(x, y) for x, y in zip(st, (crow, aux, nsl, pwin)))
        after = dump_all(eng, R, G)
        won = {int(o["gid"]): (int(e["lane"]), (int(e["bnum"]), int(e["bcoord"])))
               for o, e in zip(want, els) if int(o["verdict"]) == abi.EL_MAJORITY}
        for l in range(L):
            a = after[l]
            ex = a["coord_exists"] != 0
            assert np.array_equal(crow[l, :, 0], np.where(ex, a["coord_bnum"], 0))
            assert np.array_equal(crow[l, :, 1], np.where(ex, a["coord_bcoord"], 0))
            assert np.array_equal(crow[l, :, 2], np.where(ex, a["next_proposal_slot"], 0))
            for gid in range(G):
                touched = False
                if gid in won:
                    lane, nb = won[gid]
                    pre = crow0[l, gid]
                    higher = (pre[3] & 1) and ((int(pre[0]), int(pre[1])) > nb)  # small non-negative ballots here
                    touched = l == lane or not higher
                    if l == lane:
                        assert crow[l, gid, 3] == 3 and np.array_equal(nsl[l, :R, gid], a["node_slots"][gid, :R])
                    elif touched:
                        assert not crow[l, gid].any()
                if touched:
                    assert not pwin[l, :, gid].any()
                else:
                    assert np.array_equal(pwin[l, :, gid], pwin0[l, :, gid]) and np.array_equal(crow[l, gid], crow0[l, gid])


def test_phase1b_record_sizes_match_the_header(tmp_path):
    import os
    import subprocess
    from helpers import ROOT
    (tmp_path / "t.c").write_text('#include "gpx.h"\n#include <stdio.h>\nint main(){printf("%zu %zu %zu %zu %d %d\\n", '
                                  "sizeof(gpx_election_rec), sizeof(gpx_carryover), sizeof(gpx_election_out), "
                                  "sizeof(gpx_prepare_reply_rec), GPX_MAX_CARRY, GPX_MAX_PLAN);}\n")
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(tmp_path / "t"), str(tmp_path / "t.c")])
    out = [int(x) for x in subprocess.check_output([str(tmp_path / "t")]).decode().split()]
    assert out == [abi.election_dtype.itemsize, abi.carryover_dtype.itemsize, abi.election_out_dtype.itemsize,
                   abi.prepare_reply_dtype.itemsize, abi.GPX_MAX_CARRY, abi.GPX_MAX_PLAN] == [32, 48, 896, 288, 32, 16]


# ---- the mass case through the host mirror: one node is lost, the next one is elected in all its groups at once ---------
def drive_mass_failover(lib, batched: bool, p1b: bool = True, n_groups: int = 40):
    from gigapaxos_b200.paxos_manager import HashChainApp
    from helpers import Engine, make_config, make_requests
    NODES = [100, 101, 102]
    eng = Engine(lib, make_config(lib, max_groups=64, max_batch_recs=4096, max_batch_payload=1 << 20, checkpoint_interval=100))
    pm = PaxosManager(eng, [HashChainApp() for _ in NODES], NODES, device_phase1b=p1b)
    names = [f"TESTPaxosApp{i}" for i in range(n_groups)]
    pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
    for r in range(3):
        for n in names:
            pm.propose(n, f"{n}:{r}".encode())
        pm.run_round()
    gids = np.array([pm.instances[n].gid for n in names], dtype=np.uint32)
    rows0 = eng.dump_rows(gids, 0)
    coord = np.array([NODES.index(int(r["acc_bcoord"])) for r in rows0])
    dead = int(np.bincount(coord, minlength=3).argmax())  # the node that coordinates most groups is lost
    mine = [i for i in range(n_groups) if coord[i] == dead]
    assert len(mine) >= 5
    # before it dies its ACCEPTs for up to three more slots reach a majority, a minority, one acceptor (a gap for some)
    for k, reach in enumerate((0b011, 0b101, 0b110, 0b100)):
        sel = [i for i in mine if (i + k) % 4 != 0]  # not every group gets every slot
        if not sel:
            continue
        reqs, pay = make_requests(gids[sel], payload_len=7 + k, seed=6, round_no=k)
        reqs["flags"] = dead << 8
        reqs["entry_node"] = NODES[dead]
        acc, blob, st = eng.propose(reqs, pay)
        assert np.all(st > 0)
        acc["dst_mask"] = reach
        eng.handle_accepts(acc, blob)
    new = (dead + 1) % 3
    cand = [names[i] for i in mine]
    if batched:
        won = pm.runForCoordinators(cand + ["nonexistent"], new)
        assert won.pop("nonexistent") is False
    else:
        won = {n: pm.runForCoordinator(n, new) for n in cand}
    assert all(won.values()) and len(won) == len(mine)
    rows = [eng.dump_rows(gids[mine], l) for l in range(3)]
    assert np.all(rows[new]["coord_exists"] == 1) and np.all(rows[new]["coord_active"] == 1)
    assert np.all(rows[new]["coord_bcoord"] == NODES[new]) and not rows[dead]["coord_exists"].any()
    assert np.array_equal(rows[0]["acc_slot"], rows[1]["acc_slot"]) and np.array_equal(rows[1]["acc_slot"], rows[2]["acc_slot"])
    assert np.all(rows[0]["acc_slot"] >= rows0["acc_slot"][mine] + 1)  # the carried-over slots were decided everywhere
    s0 = pm.apps[0].state
    assert all(a.state == s0 for a in pm.apps)
    for n in names:  # business as usual under old and new coordinators
        pm.propose(n, f"{n}:after".encode(), entry_node=NODES[new])
    pm.run_round()
    pm.flush()
    assert all(a.state == pm.apps[0].state for a in pm.apps) and not pm.outstanding
    return pm


def test_mass_failover_batched_equals_one_by_one(oracle_lib):
    from test_paxos_manager import _same_end_state
    a = drive_mass_failover(oracle_lib, batched=True)
    _same_end_state(a, drive_mass_failover(oracle_lib, batched=False))
    _same_end_state(a, drive_mass_failover(oracle_lib, batched=False, p1b=False))


def test_slots_half_the_int_range_apart_do_not_run_away(oracle_lib, emu_lib):
    """a (hostile or garbage) reply pair whose recorded minimum and carried-over maximum are exactly 2^31 apart: the
    reference's fill loop `curSlot - maxCarryoverSlot <= 0` :408 would never end on it; oracle, twin and kernel count the
    slots instead and agree that there is nothing to fill"""
    R, G = 2, 4
    INT_MIN = -(1 << 31)
    eng, twin_eng = make_engine(oracle_lib, R, G), make_engine(oracle_lib, R, G)
    els = np.zeros(1, dtype=abi.election_dtype)
    els["gid"], els["lane"], els["bnum"], els["bcoord"], els["slot"], els["n_replies"] = 1, 0, 5, 100, 0, 2
    reps = np.zeros(2, dtype=abi.prepare_reply_dtype)
    reps["gid"], reps["bnum"], reps["bcoord"] = 1, 5, 100
    reps["who"] = [abi.who(0, 0), abi.who(1, 0)]
    reps["first_slot"] = -1  # gcSlot; firstSlot = 0
    reps["n_accepted"] = [0, 1]
    reps["accepted"][1][0]["slot"], reps["accepted"][1][0]["bnum"], reps["accepted"][1][0]["bcoord"] = INT_MIN, 1, 101
    reps["accepted"][1][0]["flags"] = 1 << 16
    rows = dump_all(eng, R, G)
    out = eng.handle_prepare_replies(els, reps)[0]
    # acceptor 0 records 0; acceptor 1's minimum INT_MIN is not "above" -1 and is not recorded: maxMin = 0, maxCarry = INT_MIN
    assert int(out["verdict"]) == abi.EL_MAJORITY and list(out["node_slots"][:2]) == [0, -1]
    assert int(out["n_plan"]) == 0 and int(out["next_slot"]) == INT_MIN + 1
    pm = PaxosManager(twin_eng, [NoopPaxosApp() for _ in range(R)], NODES5[:R])
    want = twin_election(pm, R, els[0], reps)
    assert out.tobytes() == want.tobytes()
    rng = np.random.default_rng(0)
    aux, crow, nsl, pwin = _state_arrays(rows, R, G, 8, R, rng)
    got = np.zeros(1, dtype=abi.election_out_dtype)
    members = np.array(NODES5[:R], dtype=np.int32)
    live = np.ones(G, dtype=np.uint8)
    assert emu_lib.emu_prepare_tally(G, R, 8, R, R, ptr(members), ptr(members), ptr(live), ptr(crow), ptr(aux), ptr(nsl), ptr(pwin),
                                     1, ptr(els), len(reps), ptr(reps), ptr(got), 64) == 1
    assert got[0].tobytes() == out.tobytes()
