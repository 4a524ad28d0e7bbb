"""GPU tests of the split lockstep record (gpx_dev.cuh, ls_rec and ls_hot): a group in lockstep keeps its ballot, aux
word and coordinator lane in a cold record that k_round_g<L, true> writes only when the group enters lockstep, and its
acc_slot, gc_slot and ns_cl in three hot planes that every in-order round writes.

Twin engines run the same calls, one with k_round_g and one with the team kernel k_round (round modes 3 and 4), and
their status, EXEC bytes, ring bytes and rows after a settle must agree byte for byte: over long runs in which the cold
records are only read, across the int32 slot wrap and slots -7..1, when groups leave lockstep for k_round_slow and
re-enter it with a new ballot and coordinator lane (so their cold records must be rewritten then), and with a lane
whose GC slot lags.
"""
import numpy as np
import pytest

from helpers import make_requests
from test_lockstep_calls_gpu import CALLS, G, oracle_twin, same_as_oracle, trio_round, view_change
from test_node_slots_compact_gpu import run_round, twins
from test_round_lockstep_gpu import compact_rounds
from test_round_parity_gpu import compare_logs
from test_round_thread_gpu import TEAM, TEAM_HOST, requests, same_rings, same_state, set_mode
from wrap_cases import NODES

pytestmark = pytest.mark.gpu

SETTLING_CALLS = ("phase_calls", "missing_decisions", "group_flags", "destroy_create", "pipeline", "kernel_timing")


@pytest.mark.parametrize("call", SETTLING_CALLS)
@pytest.mark.parametrize("L,team", [(1, TEAM), (2, TEAM), (3, TEAM), (3, TEAM_HOST)])
def test_long_lockstep_run_then_a_settling_call(cuda_lib, L, team, call):
    """twelve one-launch rounds in a row (every record stays VALID and its cold part is only read), then a call that
    settles, then three more compacting rounds"""
    a, b = twins(cuda_lib, L, G, None)
    set_mode(b, team)
    r = compact_rounds(a, b, G, L, 0, 12, one=True)
    r = CALLS[call](a, b, L, r)
    r = compact_rounds(a, b, G, L, r, 3)
    c = same_state(a, b, G, L)
    compare_logs(a, b, L)
    assert c["decisions_made"] > 15 * G
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("base", [2**31 - 5, -7])
@pytest.mark.parametrize("L", [1, 2, 3])
def test_hot_words_across_the_slot_wrap(cuda_lib, L, base):
    """slots from INT32_MAX - 5 across the wrap, and from -7 through 0 and 1: the hot slot and GC words wrap as the
    planes do; a mixed round in the middle (STOPs, absent groups, odd payload offsets) settles some records"""
    a, b = twins(cuda_lib, L, G, base)
    rng = np.random.default_rng(L + (base & 0xff))
    r = compact_rounds(a, b, G, L, 0, 5, one=True)
    run_round(a, b, G, L, r, requests(G, L, rng, r, aligned=False))
    r = compact_rounds(a, b, G, L, r + 1, 6)
    same_state(a, b, G, L)
    same_rings(a, b, L)
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("L", [1, 2, 3])
def test_leave_lockstep_and_reenter(cuda_lib, oracle_lib, L):
    """groups with VALID records leave the fast path (a second request in the batch) and write their planes back; the
    next rounds bring them back into lockstep.  Then a view change moves a subset to a new ballot and coordinator lane,
    and the records they re-enter lockstep with carry those: every later ring image and EXEC row is checked against
    the team kernel and the oracle"""
    a, b = twins(cuda_lib, L, G, None)
    eo = oracle_twin(oracle_lib, a, L, None)
    r = 0
    for _ in range(3):
        k0 = a.counters()["kernel_launches"]
        r = trio_round(a, b, eo, L, r)
        assert a.counters()["kernel_launches"] - k0 == 1
    gids = np.repeat(np.arange(G), np.where(np.arange(G) % 4 == 1, 2, 1))
    r = trio_round(a, b, eo, L, r, make_requests(gids, payload_len=1, seed=71, round_no=r, entry_lane=r % L,
                                                 entry_node=NODES[r % L]))
    launches = []
    for _ in range(4):
        k0 = a.counters()["kernel_launches"]
        r = trio_round(a, b, eo, L, r)
        launches.append(a.counters()["kernel_launches"] - k0)
    assert launches[-2:] == [1, 1], f"the groups are back on the fast path: {launches}"
    r = view_change(a, b, L, r, eo)
    for _ in range(3):
        r = trio_round(a, b, eo, L, r)
    same_as_oracle(a, eo, L)
    same_state(a, b, G, L)
    compare_logs(a, b, L)
    for e in (a, b, eo):
        e.close()


@pytest.mark.parametrize("L", [1, 2, 3])
def test_lagging_gc_slot(cuda_lib, L):
    """a lane whose acceptedGCSlot lags in a third of the groups: at L = 1 the group stays in lockstep with the
    lagging GC word in its hot plane, at L > 1 it stays on the fast path out of lockstep; four one-launch rounds with
    no settle between them, then the rows, rings and counters agree"""
    a, b = twins(cuda_lib, L, G, None)
    r = compact_rounds(a, b, G, L, 0, 3, one=True)
    gids = np.arange(0, G, 3, dtype=np.uint32)
    rows = a.dump_rows(gids, L - 1)
    assert np.array_equal(rows, b.dump_rows(gids, L - 1))
    rows["acc_gc_slot"] -= 2
    for e in (a, b):
        e.load_rows(rows)
    r = compact_rounds(a, b, G, L, r, 4, one=True)
    same_state(a, b, G, L)
    same_rings(a, b, L)
    r = compact_rounds(a, b, G, L, r, 2, one=True)
    same_state(a, b, G, L)
    for e in (a, b):
        e.close()
