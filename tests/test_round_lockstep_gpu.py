"""GPU tests of k_round_g's lockstep records: a group whose lanes advance in lockstep is kept as one 32-byte record
(gpx_dev.cuh, ls_rec) instead of its per-lane acceptor rows, coordinator row and nodeSlotNumbers word.

Twin engines run the same calls, one with k_round_g (which compacts) and one with the team kernel k_round
(gpx_set_round_mode 3, which never does).  After compacting rounds every call that reads or writes group state must
see exactly what the team engine sees: rows, rings, EXEC rows and counters are compared byte for byte (a phase
round's log and EXEC order aside).  Groups that
leave the fast path while their record is VALID are compared against the CPU oracle.
"""
import numpy as np
import pytest

from helpers import Engine, exec_by_lane, group_descs, make_config, make_requests
from test_node_slots_compact_gpu import plain_requests, raise_one, run_round, twins
from test_round_parity_gpu import compare_logs
from test_round_thread_gpu import TEAM, requests, same_rings, same_state, set_mode
from wrap_cases import NODES, SLOT_BASES

pytestmark = pytest.mark.gpu


def compact_rounds(a, b, G, L, r0, k, one=False):
    """k plain rounds from round number r0 (one: each must be one launch on the k_round_g engine)"""
    for r in range(r0, r0 + k):
        n = run_round(a, b, G, L, r)
        assert n == 1 or not one, f"round {r}: {n} launches"
    return r0 + k


def exec_set(ex):
    """EXEC records as a sorted byte set without payload_off: the phase kernels append decisions, and place bodies in
    the log, in the order their atomics ran"""
    ex = ex.copy()
    ex["payload_off"] = 0
    return np.sort(ex.view(np.uint8).reshape(-1, 24).view("V24").ravel())


def same_phase_round(a, b, reqs, pay):
    sa, xa, ea = a.round_phases(reqs, pay)
    sb, xb, eb = b.round_phases(reqs, pay)
    assert np.array_equal(sa, sb), f"status differs at {np.nonzero(sa != sb)[0][:8]}"
    assert exec_set(xa).tobytes() == exec_set(xb).tobytes(), "EXEC rows differ"
    assert exec_set(ea).tobytes() == exec_set(eb).tobytes(), "extra EXEC rows differ"


@pytest.mark.parametrize("L,base", [(1, None), (2, None), (3, None), (3, "intmax"), (2, "rs_codes")])
def test_every_state_call_after_compacting_rounds(cuda_lib, L, base):
    """compacting rounds, then each call that touches group state in turn -- dump rows, a mixed device round (STOPs,
    absent groups, odd payload offsets), the host round in phases, SET_NODE_SLOT patches, pause + unpause, the team
    kernel for one round -- each followed by more compacting rounds; both engines agree throughout"""
    G = 3001
    a, b = twins(cuda_lib, L, G, None if base is None else SLOT_BASES[base])
    rng = np.random.default_rng(17 + L)
    r = compact_rounds(a, b, G, L, 0, 3, one=True)
    same_state(a, b, G, L)  # gpx_dump_rows
    r = compact_rounds(a, b, G, L, r, 2, one=True)
    run_round(a, b, G, L, r, requests(G, L, rng, r, aligned=False))  # the VALID records of left-over groups settle
    r = compact_rounds(a, b, G, L, r + 1, 2)
    same_rings(a, b, L)  # byte for byte up to the phase round, which logs in the order its atomics ran
    same_phase_round(a, b, *plain_requests(G, L, r))
    same_state(a, b, G, L)
    r = compact_rounds(a, b, G, L, r + 1, 2)
    p = raise_one(a, G, L, np.arange(1, G, 5, dtype=np.uint32))
    assert len(p) == len(range(1, G, 5)), "every patched group has its coordinator row in the dumped planes"
    for e in (a, b):
        e.patch(p)
    run_round(a, b, G, L, r)  # the patched groups go to k_round_slow
    r = compact_rounds(a, b, G, L, r + 1, 3)
    gids = np.arange(0, G, 7, dtype=np.uint32)
    ra, pa = a.pause_groups(gids)
    rb, pb = b.pause_groups(gids)
    assert np.array_equal(pa, pb) and pa.any() and ra.tobytes() == rb.tobytes()
    for e, rows in ((a, ra), (b, rb)):
        e.load_rows(rows[pa].ravel())
    r = compact_rounds(a, b, G, L, r, 2)
    set_mode(a, TEAM)  # k_round reads the planes: settled first
    run_round(a, b, G, L, r)
    set_mode(a, 0)
    r = compact_rounds(a, b, G, L, r + 1, 2)
    c = same_state(a, b, G, L)
    compare_logs(a, b, L)
    assert c["decisions_made"] > 10 * G
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("L", [2, 3])
def test_unequal_gc_slots_stay_on_the_fast_path(cuda_lib, L):
    """a lane whose acceptedGCSlot lags keeps the group out of lockstep: it still takes the fast path (one launch per
    round), writes its planes, and agrees with the team kernel"""
    G = 2000
    a, b = twins(cuda_lib, L, G, None)
    r = compact_rounds(a, b, G, L, 0, 3, one=True)
    gids = np.arange(0, G, 3, dtype=np.uint32)
    rows = a.dump_rows(gids, L - 1)
    assert np.array_equal(rows, b.dump_rows(gids, L - 1))
    rows["acc_gc_slot"] -= 1
    for e in (a, b):
        e.load_rows(rows)
    for _ in range(4):
        assert run_round(a, b, G, L, r) == 1
        same_state(a, b, G, L)
        r += 1
    same_rings(a, b, L)
    for e in (a, b):
        e.close()


def oracle_round(eg, eo, reqs, pay, L):
    sg, xg, _ = eg.round(reqs, pay)
    so, xo, _ = eo.round(reqs, pay)
    assert np.array_equal(sg, so), f"status differs at {np.nonzero(sg != so)[0][:8]}"
    for x, y in zip(exec_by_lane(xg, L), exec_by_lane(xo, L)):  # payload_off: where each engine's log put the body
        for f in ("gid", "slot", "req_id", "flags"):
            assert np.array_equal(x[f], y[f]), f"decided (slot, request) sequence: {f}"


@pytest.mark.parametrize("L", [1, 2, 3])
def test_valid_groups_hand_off_to_the_slow_kernel(oracle_lib, cuda_lib, L):
    """after compacting rounds, groups with a second request in the batch or a STOP leave the fast path while their
    record is VALID: k_round_slow sees settled planes and the results equal the oracle's"""
    G = 1500
    kw = dict(max_groups=G, n_lanes=L, lane_node=NODES[:L], max_group_size=L, max_batch_recs=1 << 13,
              max_batch_payload=1 << 20, checkpoint_interval=4)
    eg, eo = Engine(cuda_lib, make_config(cuda_lib, **kw)), Engine(oracle_lib, make_config(oracle_lib, **kw))
    d = group_descs(G, members=NODES[:L])
    for e in (eg, eo):
        e.create_groups(d)
    for r in range(3):
        oracle_round(eg, eo, *make_requests(np.arange(G), payload_len=3, seed=5, round_no=r), L)
    gids = np.repeat(np.arange(G), np.where(np.arange(G) % 4 == 1, 2, 1))
    stop = np.zeros(len(gids), dtype=bool)
    stop[np.nonzero(gids % 9 == 4)[0]] = True
    oracle_round(eg, eo, *make_requests(gids, payload_len=3, seed=5, round_no=3, stop_mask=stop), L)
    for r in range(4, 6):
        oracle_round(eg, eo, *make_requests(np.arange(G), payload_len=3, seed=5, round_no=r), L)
    for l in range(L):
        rg, ro = eg.dump_rows(np.arange(G), l), eo.dump_rows(np.arange(G), l)
        for f in rg.dtype.names:
            assert np.array_equal(rg[f], ro[f]), f"lane {l} field {f}"
    cg, co = eg.counters(), eo.counters()
    assert cg["decisions_made"] == co["decisions_made"] and cg["stops_executed"] == co["stops_executed"] > 0
    for e in (eg, eo):
        e.close()
