"""Compact nodeSlotNumbers (ns_u, gpx_dev.cuh): a coordinator keeps one word per group while every member's entry is
equal, k_round_g reads and writes only that word and leaves a group whose entries differ to k_round_slow, and the
slow path folds the entries back into one word once they are equal again.

Twin engines run the same rounds, one with k_round_g (the default) and one with the team kernel k_round
(gpx_set_round_mode 3); their status, EXEC bytes, log rings, rows (nodeSlotNumbers included) and counters must agree
byte for byte across the transitions: SET_NODE_SLOT patches that make one member's entry differ, the rounds that bring
it back in line, the int32 slot wrap, and a pause and unpause of every group.
"""
import numpy as np
import pytest

from helpers import Engine, abi, group_descs, make_config, make_requests
from test_round_thread_gpu import NODEF, TEAM, device_round, requests, same_rings, same_state, set_mode
from wrap_cases import BALLOT_BASE, NODES, SLOT_BASES, shift_rows

pytestmark = pytest.mark.gpu


def twins(cuda_lib, L, G, base, **kw):
    """(k_round_g engine, k_round engine): G groups whose members are exactly the L lanes (all of them can take the
    in-order path), slots and ballots moved to start at `base` / BALLOT_BASE when base is not None"""
    cfg = dict(max_groups=G, n_lanes=L, lane_node=NODES[:L], window=8, max_group_size=L + 1, max_batch_recs=1 << 14,
               max_batch_payload=1 << 21, log_ring_bytes=1 << 24, checkpoint_interval=4)
    cfg.update(kw)
    es = [Engine(cuda_lib, make_config(cuda_lib, **cfg)) for _ in range(2)]
    set_mode(es[1], TEAM)
    for e in es:
        e.create_groups(group_descs(G, members=NODES[:L]))
    if base is not None:
        rows = np.concatenate([es[0].dump_rows(np.arange(G), l) for l in range(L)])
        rows = shift_rows(rows, base - int(rows["acc_slot"][0]), BALLOT_BASE)
        for e in es:
            e.load_rows(rows)
    return es


def plain_requests(G, L, r):
    """one 1-byte request per group, no STOP: every group with compact entries takes the in-order path"""
    return make_requests(np.arange(G), payload_len=1, seed=71, round_no=r, entry_lane=r % L, entry_node=NODES[r % L])


def wrap32(x):
    return int((x + 2**31) % 2**32 - 2**31)


def raise_one(e, G, L, gids):
    """SET_NODE_SLOT patches: member 1 (member 0 at L = 1) of each gid's coordinator is heard one slot ahead of the
    group's other entries, which the next in-order round catches up with"""
    m = 1 if L > 1 else 0
    out = []
    for l in range(L):
        rows = e.dump_rows(gids, l)
        for g, row in zip(gids, rows):
            if row["coord_exists"]:
                out.append((int(g), l, abi.PATCH_SET_NODE_SLOT, m, wrap32(int(row["node_slots"][m]) + 1), 0, 0, 0))
    return np.array(out, dtype=abi.patch_dtype)


def run_round(a, b, G, L, r, reqs_pay=None):
    """the same round on both engines, outputs compared; -> the kernels k_round_g's engine launched for it"""
    reqs, pay = reqs_pay if reqs_pay is not None else plain_requests(G, L, r)
    k0 = a.counters()["kernel_launches"]
    shift = 8 if r % 2 else 0
    sa, xa = device_round(a, reqs, pay, shift)
    sb, xb = device_round(b, reqs, pay, shift)
    assert np.array_equal(sa, sb), f"round {r}: status differs at {np.nonzero(sa != sb)[0][:8]}"
    assert xa.tobytes() == xb.tobytes(), f"round {r}: EXEC bytes differ at {np.nonzero(xa != xb)[0][:8]}"
    return a.counters()["kernel_launches"] - k0


@pytest.mark.parametrize("L,conf", [(1, "def"), (2, "def"), (3, "def"), (2, "nodef"), (3, "nodef")])
def test_mixed_entries_leave_and_rejoin_the_fast_path(cuda_lib, L, conf):
    """a SET_NODE_SLOT patch on a third of the groups: k_round_g leaves exactly those rounds to k_round_slow (one more
    launch), the entries are equal again after the slow round (after the next checkpoint without
    gc_majority_executed), and from then on every round is one launch again"""
    G = 3001
    a, b = twins(cuda_lib, L, G, None, **(NODEF if conf == "nodef" else {}))
    plain = run_round(a, b, G, L, 0)
    assert run_round(a, b, G, L, 1) == plain, "every group is compact after creation"
    p = raise_one(a, G, L, np.arange(0, G, 3, dtype=np.uint32))
    assert len(p) == len(range(0, G, 3)), "one coordinator lane per group"
    for e in (a, b):
        e.patch(p)
    same_state(a, b, G, L)
    launches = [run_round(a, b, G, L, r) for r in range(2, 10)]
    assert launches[0] == plain + (L > 1), "the patched groups went to k_round_slow (one member: always equal)"
    assert launches[-3:] == [plain] * 3, f"the patched groups are back on the fast path: {launches}"
    c = same_state(a, b, G, L)
    same_rings(a, b, L)
    assert c["decisions_made"] == 10 * G
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("L,conf,base", [(3, "def", "intmax"), (2, "nodef", "intmax"), (1, "def", "intmax"),
                                         (3, "def", "rs_codes")])
def test_compact_entries_across_the_slot_wrap(cuda_lib, L, conf, base):
    """in-order rounds and patched groups across the int32 slot wrap (the entries pass INT32_MAX and GPX_NS_MIXED's
    value INT32_MIN): both kernels agree byte for byte"""
    G = 1200
    a, b = twins(cuda_lib, L, G, SLOT_BASES[base], **(NODEF if conf == "nodef" else {}))
    rng = np.random.default_rng(L * 10 + len(conf))
    for r in range(8):
        if r in (1, 4):
            p = raise_one(a, G, L, np.arange(r, G, 4, dtype=np.uint32))
            for e in (a, b):
                e.patch(p)
        run_round(a, b, G, L, r, requests(G, L, rng, r, aligned=r % 2 == 0))
        same_state(a, b, G, L)
    same_rings(a, b, L)
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("L", [2, 3])
def test_compact_entries_survive_pause_and_unpause(cuda_lib, L):
    """pause every group (its rows, nodeSlotNumbers included, go to the host), restore them with load_rows -- compact
    where the entries are equal, written out where a patch made them differ -- and keep going"""
    G = 1000
    a, b = twins(cuda_lib, L, G, None)
    for r in range(2):
        run_round(a, b, G, L, r)
    p = raise_one(a, G, L, np.arange(0, G, 2, dtype=np.uint32))
    for e in (a, b):
        e.patch(p)
    gids = np.arange(G, dtype=np.uint32)
    saved = []
    for e in (a, b):
        rows, paused = e.pause_groups(gids)
        assert paused.all()
        saved.append(rows)
    assert saved[0].tobytes() == saved[1].tobytes()
    m = 1 if L > 1 else 0
    assert (saved[0]["node_slots"][0::2, :, m] != saved[0]["node_slots"][0::2, :, 0]).any(), "patched entries differ"
    for e, rows in zip((a, b), saved):
        e.load_rows(rows.reshape(-1))
    same_state(a, b, G, L)
    for r in range(2, 8):
        run_round(a, b, G, L, r)
    same_state(a, b, G, L)
    same_rings(a, b, L)
    for e in (a, b):
        e.close()
