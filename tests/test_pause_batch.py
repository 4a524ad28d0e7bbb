"""The deactivation sweep as one call (gpx_pause_groups; PaxosManager.Deactivator :2951 -> syncAndDeactivate :2806 ->
pause(Map, dequeue) :2327-2366 over PISM.tryPause :2004-2035).

CPU: the oracle's entry point against the per-group path it replaces (gpx_get_group_flags x lanes + gpx_dump_rows x lanes
+ gpx_destroy_groups), through the host mirror; and k_pause_groups' own source (gigapaxos_b200/csrc/gpx_pause.cuh)
compiled for the host (tests/emu) against the oracle.  The GPU test is in tests/test_zz_phase1b_gpu.py."""

import numpy as np
import pytest

# GPX_EMU_SANITIZE=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) python -m pytest ... : the emulated kernels under
# AddressSanitizer + UBSan (every heap buffer numpy hands them gets red zones; so do their local arrays)
from gigapaxos_b200.paxos_manager import HashChainApp, PaxosManager
from helpers import Engine, abi, emu_library, group_descs, make_config, make_requests, ptr

NODES = [100, 101, 102]


def busy_engine(lib, G=120, seed=1, journaling=1, R=3):
    """an engine whose groups are in assorted states: idle, with a commit waiting for its predecessor, with a proposal in
    flight, stopped, destroyed"""
    nodes = [100, 101, 102, 103, 104][:R]
    eng = Engine(lib, make_config(lib, n_lanes=R, lane_node=nodes, max_group_size=R, max_groups=G, max_batch_recs=4096,
                                  max_batch_payload=1 << 20, journaling_enabled=journaling))
    eng.create_groups(group_descs(G, members=tuple(nodes)))
    rng = np.random.default_rng(seed)
    gids = np.arange(G, dtype=np.uint32)
    for r in range(3):  # everybody decides three slots
        reqs, pay = make_requests(gids, payload_len=5, seed=seed, round_no=r)
        eng.round(reqs, pay)
    rows0 = eng.dump_rows(gids, 0)
    coord = np.array([nodes.index(int(x)) for x in rows0["acc_bcoord"]])
    # a third of the groups: an ACCEPT goes out but is never tallied (a proposal in flight, accepted pvalues in memory)
    sel = gids[rng.random(G) < 0.33]
    if len(sel):
        reqs, pay = make_requests(sel, payload_len=6, seed=seed, round_no=7)
        reqs["flags"] = coord[sel] << 8
        reqs["entry_node"] = np.array(nodes)[coord[sel]]
        acc, blob, st = eng.propose(reqs, pay)
        keep = rng.random(len(acc)) < 0.5
        acc["dst_mask"] = np.where(keep, (1 << R) - 1, 0b1)
        eng.handle_accepts(acc, blob)
    # a few stopped, a few destroyed
    p = np.zeros(6, dtype=abi.patch_dtype)
    p["gid"], p["lane"], p["op"], p["a"] = rng.choice(G, 6, replace=False), rng.integers(0, R, 6), abi.PATCH_SET_STATE, abi.ST_STOPPED
    eng.patch(p)
    eng.destroy_groups(rng.choice(G, 5, replace=False).astype(np.uint32))
    return eng


def per_group_pause(eng, gids):
    """what gpx_pause_groups replaces: flags and rows lane by lane, then destroy"""
    L = eng.n_lanes
    rows = np.zeros((len(gids), L), dtype=abi.row_dtype)
    ok = np.zeros(len(gids), dtype=bool)
    for i, g in enumerate(gids):
        ga = np.array([g], dtype=np.uint32)
        r = [eng.dump_rows(ga, l)[0] for l in range(L)]
        ok[i] = all(int(x["state"]) in (abi.ST_ACTIVE_1, abi.ST_ACTIVE_2) for x in r) and not any(
            int(eng.group_flags(ga, l)[0]) & abi.GF_NOT_CAUGHT_UP for l in range(L))
        if ok[i]:
            rows[i] = r
            eng.destroy_groups(ga)
    return rows, ok


@pytest.mark.parametrize("journaling,R,seed", [(1, 3, 1), (0, 3, 2), (1, 5, 3), (0, 1, 4)])
def test_oracle_pause_groups_equals_the_per_group_path(oracle_lib, journaling, R, seed):
    G = 120
    a, b = busy_engine(oracle_lib, G, seed, journaling, R), busy_engine(oracle_lib, G, seed, journaling, R)
    gids = np.random.default_rng(seed).permutation(G + 3).astype(np.uint32)  # incl. gids beyond max_groups
    gids = gids[gids < G + 3]
    rows_a, ok_a = a.pause_groups(gids)
    inb = gids < G
    rows_b, ok_b = per_group_pause(b, gids[inb])
    assert np.array_equal(ok_a[inb], ok_b) and not ok_a[~inb].any()
    assert ok_a.sum() < len(gids) and (ok_a.sum() > 0 or not journaling)  # (accepts kept in memory: the last one stays)
    assert rows_a[inb].tobytes() == rows_b.tobytes()
    for l in range(R):
        all_g = np.arange(G, dtype=np.uint32)
        assert a.dump_rows(all_g, l).tobytes() == b.dump_rows(all_g, l).tobytes()
    with pytest.raises(abi.GpxError):
        a.pause_groups(np.array([1, 2, 1], dtype=np.uint32))
    # unpause = gpx_load_rows: the paused groups come back exactly as they were dumped
    back = rows_a[ok_a].reshape(-1)
    a.load_rows(back)
    for l in range(R):
        again = a.dump_rows(gids[ok_a], l)
        for f in again.dtype.names:
            assert np.array_equal(again[f], rows_a[ok_a][:, l][f]), f


def test_mirror_pause_batch(oracle_lib):
    """PaxosManager.pauseBatch against pause() one by one: same pause table, same engine afterwards; paused instances come
    back on demand"""
    def drive(batch):
        eng = Engine(oracle_lib, make_config(oracle_lib, max_groups=64, max_batch_recs=4096, max_batch_payload=1 << 20))
        pm = PaxosManager(eng, [HashChainApp() for _ in NODES], NODES)
        names = [f"TESTPaxosApp{i}" for i in range(20)]
        pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
        for r in range(3):
            for n in names:
                pm.propose(n, f"{n}:{r}".encode())
            pm.run_round()
        pm.propose(names[3], b"queued")  # not idle: a request is waiting
        if batch:
            done = pm.pauseBatch(names[:12] + ["nonexistent", names[0]])
        else:
            done = [n for n in names[:12] if pm.pause(n)]
        assert sorted(done) == sorted(n for n in names[:12] if n != names[3])
        assert all(pm.isPaused(n) and n not in pm.instances for n in done)
        pm.run_round()
        if batch:  # half of them come back in one gpx_load_rows call, the rest on demand (propose -> unpause)
            back = pm.unpauseBatch(done[::2] + ["nonexistent"])
            assert back == done[::2] and all(not pm.isPaused(n) and n in pm.instances for n in back)
        for n in names:
            assert pm.propose(n, f"{n}:later".encode()) is not None
        pm.run_round()
        assert not pm.paused and all(a.state == pm.apps[0].state for a in pm.apps)
        return pm
    a, b = drive(True), drive(False)
    assert a.apps[0].state == b.apps[0].state and a.num_decisions == b.num_decisions


# ---- the CUDA kernels' own source on the host, driven by the engine's own sequences (gpx_state_seq.h) -------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    return emu_library(tmp_path_factory, "pause_emu")


def pause_state(eng, R, G, W, journaling, rng):
    """DevState's arrays for k_pause_groups from the oracle engine's rows and group flags, with committed / accepted
    windows synthesised so that every lane's caught-up answer is the oracle's"""
    all_g = np.arange(G, dtype=np.uint32)
    rows = [eng.dump_rows(all_g, l) for l in range(R)]
    flags = [eng.group_flags(all_g, l) for l in range(R)]
    live = (rows[0]["state"] != abi.ST_FREE).astype(np.uint8)
    acc_row = np.zeros((R, G, 4), dtype=np.int32)
    acc_aux = np.zeros((R, G), dtype=np.uint32)
    acc_win = np.zeros((R, W, G, 8), dtype=np.int32)
    coord_row = np.zeros((R, G, 4), dtype=np.int32)
    node_slots = np.zeros((R, R, G), dtype=np.int32)
    for l in range(R):
        r = rows[l]
        acc_row[l, :, 0], acc_row[l, :, 1], acc_row[l, :, 2], acc_row[l, :, 3] = r["acc_slot"], r["acc_bnum"], r["acc_bcoord"], r["acc_gc_slot"]
        busy = (flags[l] & abi.GF_NOT_CAUGHT_UP) != 0
        ex = r["coord_exists"] != 0
        # a busy lane is busy for one of the three reasons the kernel looks at (the third only without journaling)
        why = rng.integers(0, 3 if not journaling else 2, size=G)
        present = np.where(busy & ((why == 0) | ((why == 1) & ~ex)), 1 << int(rng.integers(0, 8)), 0)
        acc_aux[l] = (r["state"].astype(np.uint32) & 0xFF) | (present.astype(np.uint32) << 8) | ((flags[l].astype(np.uint32) & 3) << 24)
        outstanding = np.where(busy & (why == 1) & ex, 1 + rng.integers(0, 3, size=G), 0)
        coord_row[l, :, 0] = np.where(ex, r["coord_bnum"], 0)
        coord_row[l, :, 1] = np.where(ex, r["coord_bcoord"], 0)
        coord_row[l, :, 2] = np.where(ex, r["next_proposal_slot"], 0)
        coord_row[l, :, 3] = np.where(ex, 1 | np.where(r["coord_active"] != 0, 2, 0) | (outstanding << 8), 0)
        node_slots[l] = r["node_slots"][:, :R].T
        # accepted window: stale entries everywhere (valid but garbage-collected: slot <= gc), a live one where `why` says so
        w = int(rng.integers(0, W))
        acc_win[l, :, :, 0] = (r["acc_gc_slot"] - rng.integers(0, 3, size=G))[None, :]
        acc_win[l, :, :, 7] = 1  # GPX_ENT_VALID
        livepv = busy & (why == 2)
        acc_win[l, w, :, 0] = np.where(livepv, r["acc_gc_slot"] + 1 + rng.integers(0, 4, size=G), acc_win[l, w, :, 0])
    return live, acc_row, acc_aux, acc_win, coord_row, node_slots


@pytest.mark.parametrize("journaling,R,seed,block", [(1, 3, 5, 128), (0, 3, 6, 1), (1, 5, 7, 33), (0, 2, 8, 128)])
def test_kernel_source_on_the_host_equals_oracle(oracle_lib, emu_lib, journaling, R, seed, block):
    """DevState's arrays are filled from the oracle engine's rows and group flags (committed / accepted windows are
    synthesised so that every lane's caught-up answer is the oracle's), k_pause_groups runs thread by thread, and its
    verdicts, rows and the state it leaves are the oracle's."""
    G, W = 120, 8
    nodes = [100, 101, 102, 103, 104][:R]
    # (the oracle engine journals either way: with accepts kept in memory its last accepted pvalue never leaves and nothing
    # pauses.  `journaling` here is the KERNEL's flag -- 0 makes it look through the synthesised accepted windows too)
    eng = busy_engine(oracle_lib, G, seed, 1, R)
    all_g = np.arange(G, dtype=np.uint32)
    rng = np.random.default_rng(seed)
    live, acc_row, acc_aux, acc_win, coord_row, node_slots = pause_state(eng, R, G, W, journaling, rng)
    gids = rng.permutation(G + 2).astype(np.uint32)
    want_rows, want_ok = eng.pause_groups(gids)
    got_rows = np.zeros((len(gids), R), dtype=abi.row_dtype)
    got_ok = np.full(len(gids), 7, dtype=np.uint8)
    nodes_a = np.array(nodes, dtype=np.int32)
    rc = emu_lib.emu_pause_groups(G, R, W, R, R, ptr(nodes_a), ptr(nodes_a), ptr(live), int(journaling), ptr(acc_row), ptr(acc_aux),
                                  ptr(acc_win), ptr(coord_row), ptr(node_slots), len(gids), ptr(gids), ptr(got_rows), ptr(got_ok),
                                  block)
    assert rc == 1
    assert np.array_equal(got_ok.astype(bool), want_ok) and 0 < want_ok.sum() < len(gids)
    for f in got_rows.dtype.names:
        if f in ("version", "name_hash"):  # kept on the host by the engine (gpx_dump_rows fills them in)
            continue
        assert np.array_equal(got_rows[f][want_ok], want_rows[f][want_ok]), f
    assert not got_rows[~want_ok].view(np.uint8).any()  # rows of groups that did not pause are not written
    # a gid twice in the batch: refused before anything runs
    aux0, rows0 = acc_aux.copy(), got_rows.copy()
    dup = np.array([gids[0], gids[1], gids[0]], dtype=np.uint32)
    assert emu_lib.emu_pause_groups(G, R, W, R, R, ptr(nodes_a), ptr(nodes_a), ptr(live), int(journaling), ptr(acc_row),
                                    ptr(acc_aux), ptr(acc_win), ptr(coord_row), ptr(node_slots), len(dup), ptr(dup),
                                    ptr(got_rows), ptr(got_ok), block) == abi.GPX_EINVAL
    assert b"twice" in emu_lib.emu_last_error() and np.array_equal(acc_aux, aux0) and np.array_equal(got_rows, rows0)
    after = [eng.dump_rows(all_g, l) for l in range(R)]
    for l in range(R):
        freed = after[l]["state"] == abi.ST_FREE
        assert np.array_equal(acc_aux[l] & 0xFF, after[l]["state"].astype(np.uint32) & 0xFF)
        assert np.array_equal(acc_row[l, :, 0][~freed], after[l]["acc_slot"][~freed])
        assert np.all(acc_row[l][freed] == np.array([0, -1, -1, -1])) and not coord_row[l][freed].any()


# ---- gpx_select_groups: which groups a sweep has to look at --------------------------------------------------------------
@pytest.mark.parametrize("R,seed", [(3, 11), (5, 12)])
def test_oracle_select_groups_equals_the_per_group_flags(oracle_lib, R, seed):
    G = 120
    eng = busy_engine(oracle_lib, G, seed, 1, R)
    all_g = np.arange(G, dtype=np.uint32)
    for lane in range(R):
        rows, flags = eng.dump_rows(all_g, lane), eng.group_flags(all_g, lane)
        active = np.isin(rows["state"], (abi.ST_ACTIVE_1, abi.ST_ACTIVE_2))
        for mask, value in ((abi.GF_NOT_CAUGHT_UP, 0), (abi.GF_NOT_CAUGHT_UP, abi.GF_NOT_CAUGHT_UP), (0, 0),
                            (abi.GF_NEEDS_SYNC, abi.GF_NEEDS_SYNC)):
            want = all_g[active & ((flags & mask) == value)]
            assert np.array_equal(eng.select_groups(lane, mask, value), want)
        n_idle = int((active & ((flags & abi.GF_NOT_CAUGHT_UP) == 0)).sum())
        assert 0 < n_idle < G
        with pytest.raises(abi.GpxError):
            eng.select_groups(lane, abi.GF_NOT_CAUGHT_UP, 0, cap=n_idle - 1)  # more matches than the buffer holds


def test_mirror_sync_and_deactivate(oracle_lib):
    """PaxosManager.syncAndDeactivate: the engine names the groups; idle ones are paused in one batch and come back on
    demand"""
    eng = Engine(oracle_lib, make_config(oracle_lib, max_groups=64, max_batch_recs=4096, max_batch_payload=1 << 20))
    pm = PaxosManager(eng, [HashChainApp() for _ in NODES], NODES)
    names = [f"TESTPaxosApp{i}" for i in range(24)]
    pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
    for r in range(2):
        for n in names:
            pm.propose(n, f"{n}:{r}".encode())
        pm.run_round()
    pm.propose(names[5], b"waiting")  # queued at the host: not idle
    res = pm.syncAndDeactivate()
    assert res == {"synced": 0, "paused": 23} and not pm.isPaused(names[5])
    assert len(eng.select_groups(0, 0, 0)) == 1
    pm.run_round()
    for n in names:
        assert pm.propose(n, b"again") is not None
    pm.run_round()
    assert not pm.paused and all(a.state == pm.apps[0].state for a in pm.apps)


@pytest.mark.parametrize("journaling,R,seed,block", [(1, 3, 21, 128), (0, 5, 22, 7)])
def test_select_kernel_source_on_the_host_equals_oracle(oracle_lib, emu_lib, journaling, R, seed, block):
    """k_select_groups on the state arrays of test_kernel_source_on_the_host_equals_oracle above"""
    G, W = 120, 8
    nodes = [100, 101, 102, 103, 104][:R]
    eng = busy_engine(oracle_lib, G, seed, 1, R)
    all_g = np.arange(G, dtype=np.uint32)
    rows = [eng.dump_rows(all_g, l) for l in range(R)]
    flags = [eng.group_flags(all_g, l) for l in range(R)]
    rng = np.random.default_rng(seed)
    live = (rows[0]["state"] != abi.ST_FREE).astype(np.uint8)
    acc_row = np.zeros((R, G, 4), dtype=np.int32)
    acc_aux = np.zeros((R, G), dtype=np.uint32)
    acc_win = np.zeros((R, W, G, 8), dtype=np.int32)
    coord_row = np.zeros((R, G, 4), dtype=np.int32)
    for l in range(R):
        r = rows[l]
        acc_row[l, :, 3] = r["acc_gc_slot"]
        busy = (flags[l] & abi.GF_NOT_CAUGHT_UP) != 0
        ex = r["coord_exists"] != 0
        why = rng.integers(0, 3 if not journaling else 2, size=G)
        present = np.where(busy & ((why == 0) | ((why == 1) & ~ex)), 1 << int(rng.integers(0, 8)), 0)
        sticky = rng.integers(0, 4, size=G).astype(np.uint32)  # OVERFLOW / NEEDS_SYNC bits
        acc_aux[l] = (r["state"].astype(np.uint32) & 0xFF) | (present.astype(np.uint32) << 8) | (sticky << 24)
        coord_row[l, :, 3] = np.where(ex, 1 | (np.where(busy & (why == 1), 2, 0) << 8), 0)
        acc_win[l, :, :, 0] = (r["acc_gc_slot"] - 1)[None, :]
        acc_win[l, :, :, 7] = 1
        livepv = busy & (why == 2)
        acc_win[l, 3, :, 0] = np.where(livepv, r["acc_gc_slot"] + 2, acc_win[l, 3, :, 0])
        flags[l] = (flags[l] & abi.GF_NOT_CAUGHT_UP) | sticky.astype(np.uint8)
    nodes_a = np.array(nodes, dtype=np.int32)
    for lane in range(R):
        active = np.isin(rows[lane]["state"], (abi.ST_ACTIVE_1, abi.ST_ACTIVE_2))
        for mask, value in ((abi.GF_NOT_CAUGHT_UP, 0), (abi.GF_NEEDS_SYNC, abi.GF_NEEDS_SYNC),
                            (abi.GF_NEEDS_SYNC | abi.GF_NOT_CAUGHT_UP, abi.GF_NOT_CAUGHT_UP), (0, 0)):
            want = all_g[active & ((flags[lane] & mask) == value)]
            for cap, spec in ((G, b"asc"), (G, b"desc"), (max(len(want) - 2, 0), b"desc")):
                out = np.full(max(cap, 1), 0xFFFFFFFF, dtype=np.uint32)
                found = np.zeros(1, dtype=np.uint32)
                emu_lib.emu_set_order(spec)  # the kernel appends in thread order; the host sorts what it appended
                rc = emu_lib.emu_select_groups(G, R, W, R, R, ptr(nodes_a), ptr(nodes_a), ptr(live), int(journaling), ptr(acc_row),
                                               ptr(acc_aux), ptr(acc_win), ptr(coord_row), lane, mask, value, ptr(out), cap,
                                               ptr(found), block)
                emu_lib.emu_set_order(None)
                assert rc == 1 and int(found[0]) == len(want)
                got = out[: min(cap, len(want))]  # sorted on the host
                assert np.array_equal(got, want) if cap >= len(want) else np.all(np.isin(got, want))
                assert np.all(np.diff(got.astype(np.int64)) > 0) and np.all(out[len(got):] == 0xFFFFFFFF)


# ---- the slow-path list end to end: a replica that missed decisions is named by the engine, caught up, taken off the list ---
def drive_flagged_sync(lib):
    from gigapaxos_b200.paxos_manager import RequestPacket
    eng = Engine(lib, make_config(lib, max_groups=64, max_batch_recs=4096, max_batch_payload=1 << 20, checkpoint_interval=100))
    pm = PaxosManager(eng, [HashChainApp() for _ in NODES], NODES)
    names = [f"TESTPaxosApp{i}" for i in range(6)]
    pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
    for r in range(2):
        for n in names:
            pm.propose(n, f"{n}:{r}".encode())
        pm.run_round()
    gids = np.array([pm.instances[n].gid for n in names], dtype=np.uint32)
    rows0 = eng.dump_rows(gids, 0)
    coord = [NODES.index(int(rows0[i]["acc_bcoord"])) for i in range(len(names))]
    for k in range(11):  # lane 2 is cut off for 11 slots (more than the window), then hears the LAST decision only
        reqs, pay = make_requests(gids, payload_len=5 + k % 7, seed=9, round_no=k)
        reqs["flags"] = [c << 8 for c in coord]
        reqs["entry_node"] = [NODES[c] for c in coord]
        acc, blob, st = eng.propose(reqs, pay)
        assert np.all(st > 0)
        acc["dst_mask"] = 0b011
        rep, _ = eng.handle_accepts(acc, blob)
        dec = eng.handle_accept_replies(rep)
        dec["dst_mask"] = 0b111 if k == 10 else 0b011
        ex, extra = eng.handle_decisions(dec)
        batches = {int(r["req_id"]): [RequestPacket(names[i], int(r["req_id"]),
                                                    bytes(pay[int(r["payload_off"]): int(r["payload_off"]) + int(r["payload_len"])]),
                                                    entry_replica=NODES[coord[i]])] for i, r in enumerate(reqs)}
        pm._apply(np.concatenate([ex, extra]), batches)
    listed = eng.select_groups(2, abi.GF_NEEDS_SYNC, abi.GF_NEEDS_SYNC)
    assert np.array_equal(listed, np.sort(gids)) and len(eng.select_groups(0, abi.GF_NEEDS_SYNC, abi.GF_NEEDS_SYNC)) == 0
    assert pm.apps[2].state != pm.apps[0].state
    res = pm.syncAndDeactivate(pause=False)
    assert res["synced"] == 11 * len(names) and pm.apps[2].state == pm.apps[0].state
    assert len(eng.select_groups(2, abi.GF_NEEDS_SYNC, abi.GF_NEEDS_SYNC)) == 0  # dealt with: off the list
    assert pm.syncAndDeactivate(pause=False) == {"synced": 0, "paused": 0}
    return pm


def test_slow_path_list_end_to_end(oracle_lib):
    drive_flagged_sync(oracle_lib)


# ---- gpx_missing_decisions: the fields of a SYNC_DECISIONS_REQUEST ------------------------------------------------------------
def engine_with_holes(lib):
    """lane 2 of every group: slot s gets no commit, s+1 a commit without its accept, s+2 commit and accept, s+3 the last
    commit (groups 0..9); groups 10..19 are fully caught up; group 20's lane 2 is stopped"""
    G = 24
    eng = Engine(lib, make_config(lib, max_groups=G, max_batch_recs=4096, max_batch_payload=1 << 20, checkpoint_interval=100))
    eng.create_groups(group_descs(G))
    gids = np.arange(G, dtype=np.uint32)
    for r in range(2):
        reqs, pay = make_requests(gids, payload_len=4, seed=2, round_no=r)
        eng.round(reqs, pay)
    rows0 = eng.dump_rows(gids, 0)
    coord = np.array([NODES.index(int(x)) for x in rows0["acc_bcoord"]])
    sel = gids[:10][coord[:10] != 2]  # (a coordinator on lane 2 would see its own proposals)
    for k in range(4):
        reqs, pay = make_requests(sel, payload_len=5, seed=3, round_no=k)
        reqs["flags"] = coord[sel] << 8
        reqs["entry_node"] = np.array(NODES)[coord[sel]]
        acc, blob, st = eng.propose(reqs, pay)
        acc["dst_mask"] = 0b111 if k >= 2 else 0b011  # lane 2 hears the accepts of s+2, s+3 only
        rep, _ = eng.handle_accepts(acc, blob)
        dec = eng.handle_accept_replies(rep)
        dec["dst_mask"] = 0b111 if k >= 1 else 0b011  # ... and the commits of s+1, s+2, s+3
        eng.handle_decisions(dec)
    p = np.zeros(1, dtype=abi.patch_dtype)
    p["gid"], p["lane"], p["op"], p["a"] = 20, 2, abi.PATCH_SET_STATE, abi.ST_STOPPED
    eng.patch(p)
    return eng, sel


def test_oracle_missing_decisions(oracle_lib):
    eng, sel = engine_with_holes(oracle_lib)
    all_g = np.arange(26, dtype=np.uint32)  # incl. two gids that do not exist
    m = eng.missing_decisions(2, all_g)
    rows = eng.dump_rows(all_g[:24], 2)
    for g in sel:
        r, s = m[g], int(rows[g]["acc_slot"])
        assert int(r["slot"]) == s and int(r["max_decision_slot"]) == s + 3
        assert list(r["missing"][: int(r["n_missing"])]) == [s, s + 1]  # no commit; a commit without its accept
        assert not r["missing_too_much"] and int(r["flags"]) & abi.GF_NOT_CAUGHT_UP
    for g in range(10, 20):
        r, s = m[g], int(rows[g]["acc_slot"])
        assert int(r["max_decision_slot"]) == s - 1 and list(r["missing"][: int(r["n_missing"])]) == [s]  # :2297-2298
    assert int(m[20]["n_missing"]) == 0 and int(m[20]["max_decision_slot"]) == int(rows[20]["acc_slot"]) - 1  # stopped
    assert int(m[24]["n_missing"]) == 0 and int(m[25]["slot"]) == 0
    lim = eng.missing_decisions(2, sel, size_limit=1)
    assert all(list(r["missing"][: int(r["n_missing"])]) == [int(r["slot"])] for r in lim)  # sizeLimit cuts the list
    few = eng.missing_decisions(2, sel, too_much_gap=3)
    assert all(r["missing_too_much"] for r in few)  # a gap of 3 >= the threshold
    # the SYNC_DECISIONS packet built from a record
    from gigapaxos_b200 import packets_json as pj
    r = m[sel[0]]
    pkt = pj.sync_decisions_json("NoopPaxosApp%d" % sel[0], 0, 102, int(r["max_decision_slot"]), r["missing"][: int(r["n_missing"])])
    assert pj.parse_packet(pkt)["missing"] == [int(r["slot"]), int(r["slot"]) + 1]


def model_missing(slot, gc, state, present, valued, win, W, size_limit, gap_th):
    """PaxosAcceptor.getMaxCommittedSlot / getMissingCommittedSlots / PISM.isMissingTooMuch on one lane's window, in Python"""
    i32 = lambda v: ((int(v) + (1 << 31)) % (1 << 32)) - (1 << 31)
    max_c = i32(slot - 1)
    if state != abi.ST_STOPPED:
        for d in range(W):
            s = i32(slot + d)
            if (present >> (s & (W - 1))) & 1:
                max_c = s
    missing = []
    if state in (abi.ST_ACTIVE_1, abi.ST_ACTIVE_2):
        for d in range(W):
            s = i32(slot + d)
            if not (i32(s - max_c) < 0 and i32(s - i32(slot + size_limit)) < 0):
                break
            w = s & (W - 1)
            if not (present >> w) & 1:
                missing.append(s)
            elif not (valued >> w) & 1:
                e = win[w]
                if not ((e[7] & 1) and e[0] == s and i32(s - gc) > 0):
                    missing.append(s)
        if not missing:
            missing = [slot]
        gap = i32(max_c - slot)
        too = gap >= gap_th or (slot in (0, 1) and (gap >= int(gap_th / 100) or gap_th <= 1))
    else:
        too = False
    return max_c, missing, too


@pytest.mark.parametrize("seed,block,wrap", [(31, 128, False), (32, 5, True)])
def test_missing_kernel_source_on_the_host_equals_the_model(emu_lib, seed, block, wrap):
    rng = np.random.default_rng(seed)
    G, L, W, R = 200, 3, 8, 3
    base = 0x7FFFFFF0 if wrap else 0
    i32 = lambda v: ((int(v) + (1 << 31)) % (1 << 32)) - (1 << 31)
    live = (rng.random(G) < 0.9).astype(np.uint8)
    acc_row = np.zeros((L, G, 4), dtype=np.int32)
    acc_aux = np.zeros((L, G), dtype=np.uint32)
    acc_win = np.zeros((L, W, G, 8), dtype=np.int32)
    coord_row = np.zeros((L, G, 4), dtype=np.int32)
    for l in range(L):
        for g in range(G):
            slot = i32(base + int(rng.integers(0, 40)))
            gc = i32(slot - int(rng.integers(1, 6)))
            state = int(rng.choice([abi.ST_ACTIVE_1, abi.ST_ACTIVE_1, abi.ST_ACTIVE_2, abi.ST_STOPPED, abi.ST_RECOVERY]))
            present = int(rng.integers(0, 256)) if rng.random() < 0.7 else 0
            valued = present & int(rng.integers(0, 256))
            acc_row[l, g] = [slot, 1, 100, gc]
            acc_aux[l, g] = state | (present << 8) | (valued << 16) | (int(rng.integers(0, 4)) << 24)
            for w in range(W):
                k = int(rng.integers(0, 4))  # the accept of the slot that maps here / of an older lap / invalid / below gc
                s = next(i32(slot + d) for d in range(W) if (i32(slot + d) & (W - 1)) == w)
                acc_win[l, w, g, 0] = [s, i32(s - W), s, i32(gc - 1)][k]
                acc_win[l, w, g, 7] = 0 if k == 2 else 1
    gids = rng.permutation(G + 3).astype(np.uint32)
    nodes = np.array(NODES, dtype=np.int32)
    for lane in range(L):
        for size_limit, gap_th in ((400, 400), (3, 400), (400, 4), (400, 1)):
            out = np.zeros(len(gids), dtype=abi.missing_dtype)
            out.view(np.uint8)[:] = 0x5A
            assert emu_lib.emu_missing_decisions(G, L, W, R, ptr(nodes), ptr(nodes), ptr(live), 1, ptr(acc_row), ptr(acc_aux),
                                                 ptr(acc_win), ptr(coord_row), lane, len(gids), ptr(gids), size_limit, gap_th,
                                                 ptr(out), block) == 1
            for r, g in zip(out, gids):
                assert int(r["gid"]) == g
                if g >= G or not live[g]:
                    assert int(r["n_missing"]) == 0 and int(r["slot"]) == 0 and not r["missing"].any()
                    continue
                slot, gc = int(acc_row[lane, g, 0]), int(acc_row[lane, g, 3])
                aux = int(acc_aux[lane, g])
                max_c, missing, too = model_missing(slot, gc, aux & 0xFF, (aux >> 8) & 0xFF, (aux >> 16) & 0xFF,
                                                    acc_win[lane, :, g], W, size_limit, gap_th)
                assert int(r["slot"]) == slot and int(r["max_decision_slot"]) == max_c, (lane, g)
                assert list(r["missing"][: int(r["n_missing"])]) == missing and bool(r["missing_too_much"]) == too, (lane, g)
                assert not r["missing"][int(r["n_missing"]):].any()


@pytest.mark.parametrize("seed,block", [(41, 128), (42, 3)])
def test_clear_flags_kernel_source_on_the_host(emu_lib, seed, block):
    """gpx_clear_group_flags: only the OVERFLOW / NEEDS_SYNC bits of the mask, only this lane, only these gids (those
    beyond max_groups are skipped); a gid twice or a lane beyond the engine's is refused and nothing changes"""
    rng = np.random.default_rng(seed)
    G, L, W, R = 150, 3, 8, 3
    nodes = np.array(NODES, dtype=np.int32)
    live = np.ones(G, dtype=np.uint8)
    aux = rng.integers(0, 1 << 32, size=(L, G), dtype=np.uint64).astype(np.uint32)
    for lane in range(L):
        for mask in (abi.GF_NEEDS_SYNC, abi.GF_OVERFLOW | abi.GF_NEEDS_SYNC | abi.GF_NOT_CAUGHT_UP, 0):
            gids = rng.choice(G + 5, size=60, replace=False).astype(np.uint32)
            want = aux.copy()
            ok = gids[gids < G]
            want[lane, ok] &= ~np.uint32((mask & (abi.GF_OVERFLOW | abi.GF_NEEDS_SYNC)) << 24)
            assert emu_lib.emu_clear_group_flags(G, L, W, R, ptr(nodes), ptr(nodes), ptr(live), ptr(aux), lane,
                                                 len(gids), ptr(gids), mask, block) == 0
            assert np.array_equal(aux, want)
    before = aux.copy()
    dup = np.array([4, 9, 4], dtype=np.uint32)
    assert emu_lib.emu_clear_group_flags(G, L, W, R, ptr(nodes), ptr(nodes), ptr(live), ptr(aux), 0, 3, ptr(dup),
                                         abi.GF_NEEDS_SYNC, block) == abi.GPX_EINVAL
    assert b"twice" in emu_lib.emu_last_error()
    assert emu_lib.emu_clear_group_flags(G, L, W, R, ptr(nodes), ptr(nodes), ptr(live), ptr(aux), L, 2, ptr(dup),
                                         abi.GF_NEEDS_SYNC, block) == abi.GPX_ERANGE
    assert np.array_equal(aux, before)
