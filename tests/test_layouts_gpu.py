"""GPU parity against the oracle in every engine layout: 1 to 8 lanes in any order, groups of 1 to 16 members with lanes
outside the group and remote members (tests/layout_cases.py).  Everything is compared bit-exactly, as in the other
parity tests: status, ACCEPT / reply / DECISION / EXEC records, rows of every lane, counters, log ring bytes.

  - every layout under the adversarial schedules of tests/fuzz.py: the phase calls, k_act, gpx_round or
    gpx_round_phases, PREPAREs, view changes, remote members' replies;
  - in-order rounds of G = 3001 identity groups (a partial last warp) at every lane count 1-8: one launch per round
    (the in-order fast path took every group), full and compact output;
  - the compact nodeSlotNumbers (ns_u) at L > 3 and R != L: SET_NODE_SLOT patches, a view change through
    gpx_handle_prepare_replies, a lagging member's ACCEPT_REPLY, pause and unpause;
  - the input rules: duplicate lane nodes and members, group sizes, the 4096-set limit, and a refused call that
    introduced a member set followed by one that uses it.
"""
import numpy as np
import pytest

from fuzz import Fuzzer
from helpers import Engine, abi, canon, exec_by_lane, group_descs, make_config, make_requests
from layout_cases import (LAYOUTS, MAX_MSETS, N8, assert_reached, check_input_rules, descs, mset_limit_engine,
                          refused, small_engine)
from p1b_cases import assert_same_out, assert_same_rows, make_engine, preconditions, random_elections
from test_node_slots_compact_gpu import raise_one
from test_round_parity_gpu import compare_logs

pytestmark = pytest.mark.gpu


def same_state(eo, eg, G):
    """rows of every lane (of a gid never created, only the state FREE), counters"""
    gids = np.arange(G)
    for lane in range(eg.n_lanes):
        ro, rg = eo.dump_rows(gids, lane), eg.dump_rows(gids, lane)
        assert np.array_equal(ro["state"], rg["state"]), f"lane {lane}: state"
        live = ro["state"] != abi.ST_FREE
        ro, rg = ro[live], rg[live]
        assert ro.tobytes() == rg.tobytes(), f"rows of lane {lane} differ at gids {ro['gid'][ro != rg][:8]}"
    co, cg = eo.counters(), eg.counters()
    co.pop("kernel_launches"), cg.pop("kernel_launches")
    assert co == cg, {k: (co[k], cg[k]) for k in co if co[k] != cg[k]}
    return co


def same_round(eo, eg, reqs, pay, fn="round"):
    """one round on both engines: status, the EXEC records of every lane (in gid order), the extra executions as a
    set; -> (oracle status, the kernels the device launched)"""
    k0 = eg.counters()["kernel_launches"]
    cap = 4 * len(reqs) * eg.n_lanes + 256
    so, xo, to = getattr(eo, fn)(reqs, pay, extra_cap=cap)
    sg, xg, tg = getattr(eg, fn)(reqs, pay, extra_cap=cap)
    launches = eg.counters()["kernel_launches"] - k0
    assert np.array_equal(so, sg), f"status differs at {np.nonzero(so != sg)[0][:8]}"
    for lane, (a, b) in enumerate(zip(exec_by_lane(np.concatenate([xo, to]), eg.n_lanes),
                                      exec_by_lane(np.concatenate([xg, tg]), eg.n_lanes))):
        a, b = a[np.lexsort((a["slot"], a["gid"]))], b[np.lexsort((b["slot"], b["gid"]))]
        assert len(a) == len(b), f"lane {lane}: {len(a)} vs {len(b)} executions"
        single = (a["flags"] >> 16) <= 1  # a BATCHED blob's log position depends on block scheduling
        for f in a.dtype.names:
            x, y = (a[f][single], b[f][single]) if f == "payload_off" else (a[f], b[f])
            assert np.array_equal(x, y), f"lane {lane}: exec {f}"
    return so, launches


# ---- every layout under adversarial schedules -------------------------------------------------------------------------

@pytest.mark.parametrize("fn", ["round", "round_phases"])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_layout_parity(oracle_lib, cuda_lib, name, fn):
    seed = 1000 + sorted(LAYOUTS).index(name) * 2 + (fn == "round_phases")
    f = Fuzzer([oracle_lib, cuda_lib], G=128, W=8, seed=seed, **LAYOUTS[name])
    assert f.run(steps=40, check_every=5, fused_prob=0.3, round_prob=0.4, round_fn=fn, prepares=True) > 100
    assert_reached(f, name)
    compare_logs(f.engines[0], f.engines[1], f.L)
    f.close()


# ---- in-order identity rounds at every lane count --------------------------------------------------------------------

def identity_pair(oracle_lib, cuda_lib, L, G, lane_node=None, members=None, **kw):
    nodes = N8[:L] if lane_node is None else lane_node
    cfg = dict(max_groups=G, n_lanes=L, lane_node=nodes, max_group_size=max(L, 3), max_batch_recs=4096,
               max_batch_payload=1 << 20, log_ring_bytes=1 << 24, checkpoint_interval=3)
    cfg.update(kw)
    eo, eg = Engine(oracle_lib, make_config(oracle_lib, **cfg)), Engine(cuda_lib, make_config(cuda_lib, **cfg))
    d = group_descs(G, members=N8[:L]) if members is None else descs([members[g % len(members)] for g in range(G)])
    for e in (eo, eg):
        e.create_groups(d)
    return eo, eg


def plain(G, L, r, nodes=N8):
    return make_requests(np.arange(G), payload_len=1 + 5 * (r % 4), seed=91, round_no=r, entry_lane=r % L,
                         entry_node=nodes[r % L])


@pytest.mark.parametrize("L", [1, 2, 3, 4, 5, 6, 7, 8])
def test_in_order_identity_rounds(oracle_lib, cuda_lib, L):
    """every group takes the in-order path of k_round_g (L <= 3) or the team kernel k_round (L > 3; 32 mod L lanes of
    a warp idle at L = 5, 6, 7): one launch per round, in full and in compact output mode"""
    G = 3001
    eo, eg = identity_pair(oracle_lib, cuda_lib, L, G)
    for r in range(4):
        reqs, pay = plain(G, L, r)
        st, launches = same_round(eo, eg, reqs, pay)
        assert launches == 1, f"round {r}: {launches} launches"
        assert np.all(st == r + 1)
    for r in range(4, 7):  # compact summaries: every lane executed the request in order
        reqs, pay = plain(G, L, r)
        k0 = eg.counters()["kernel_launches"]
        out = eg.round_wait(eg.round_submit(reqs, pay, compact=True, extra_cap=G * L + 64))
        assert eg.counters()["kernel_launches"] - k0 == 1
        so, xo, to = eo.round(reqs, pay)
        assert len(to) == 0 and out["n_extra"] == 0
        s = out["sum"]
        assert np.array_equal(s["slot"], so)
        assert np.all(s["lane_mask"] == (1 << L) - 1) and np.all(s["nreq"] == 1)
        x0 = exec_by_lane(xo, L)[0]
        assert np.array_equal(x0["gid"], np.arange(G))
        assert np.array_equal(s["flags"], (x0["flags"] & abi.F_CKPT).astype(np.uint8))
    c = same_state(eo, eg, G)
    assert c["decisions_made"] == 7 * G and c["executed"] == 7 * G * L and c["checkpoints_due"] > 0
    compare_logs(eo, eg, L)
    for e in (eo, eg):
        e.close()


# ---- compact nodeSlotNumbers at L > 3 and R != L ---------------------------------------------------------------------

NS_LAYOUTS = {  # (lane_node, members)
    "ident5": (N8[:5], [N8[:5]]),
    "sub4of6": ([105, 101, 100, 103, 102, 104], [N8[:6], N8[1:5]]),
    "sub3of8": (N8, [N8, [100, 102, 104], [101, 103, 105, 107]]),
}


def at_members(G, r, lane_node, members):
    """one request per group, entering at member r mod R of its group (a lane outside the group has no instance)"""
    reqs, pay = plain(G, len(lane_node), r, lane_node)
    ms = [members[g % len(members)] for g in range(G)]
    nodes = np.array([m[r % len(m)] for m in ms])
    reqs["flags"] = np.array([lane_node.index(n) for n in nodes], dtype=np.uint32) << 8
    reqs["entry_node"] = nodes
    return reqs, pay


@pytest.mark.parametrize("name", sorted(NS_LAYOUTS))
def test_node_slots_patch_lag_and_pause(oracle_lib, cuda_lib, name):
    """SET_NODE_SLOT patches make one member's entry differ; a member that missed an ACCEPT acks it late (its reply
    carries an older maxCheckpointedSlot); every group is paused and restored; in-order rounds between each step --
    against the oracle, byte for byte"""
    lane_node, members = NS_LAYOUTS[name]
    L, G = len(lane_node), 1200
    eo, eg = identity_pair(oracle_lib, cuda_lib, L, G, lane_node, members, max_group_size=8)
    for r in range(2):
        same_round(eo, eg, *at_members(G, r, lane_node, members))
    p = raise_one(eg, G, L, np.arange(0, G, 3, dtype=np.uint32))
    assert len(p) > G // 4
    for e in (eo, eg):
        e.patch(p)
    same_state(eo, eg, G)
    for r in range(2, 6):
        same_round(eo, eg, *at_members(G, r, lane_node, members))
    same_state(eo, eg, G)
    # a lagging member: the ACCEPTs of one round miss the last member lane of every group, reach it after the decisions
    reqs, pay = at_members(G, 6, lane_node, members)
    (ao, bo, so), (ag, bg, sg) = eo.propose(reqs, pay), eg.propose(reqs, pay)
    assert np.array_equal(so, sg)
    ao, ag = canon(ao), canon(ag)
    assert len(ao) == len(ag) > G // 2
    for f in ("gid", "slot", "bnum", "dst_mask", "req_id"):  # payload_off is each side's own
        assert np.array_equal(ao[f], ag[f]), f"propose: {f}"
    lag = np.array([1 << (int(m).bit_length() - 1) for m in ao["dst_mask"]], dtype=np.uint16)
    for a in (ao, ag):
        a["dst_mask"] = a["dst_mask"] & ~lag
    rep = [e.handle_accepts(a, b)[0] for e, a, b in ((eo, ao, bo), (eg, ag, bg))]
    assert canon(rep[0]).tobytes() == canon(rep[1]).tobytes()
    dec = [e.handle_accept_replies(canon(x)) for e, x in zip((eo, eg), rep)]
    assert canon(dec[0]).tobytes() == canon(dec[1]).tobytes() and len(dec[0]) == len(ao)
    for e, d in zip((eo, eg), dec):
        e.handle_decisions(canon(d))
    for a in (ao, ag):
        a["dst_mask"] = lag
    rep = [e.handle_accepts(a, b)[0] for e, a, b in ((eo, ao, bo), (eg, ag, bg))]
    late = canon(rep[0])
    assert late.tobytes() == canon(rep[1]).tobytes() and len(late) == len(ao)
    dec = [e.handle_accept_replies(late) for e in (eo, eg)]
    assert dec[0].tobytes() == dec[1].tobytes()
    same_state(eo, eg, G)
    for r in range(7, 10):
        same_round(eo, eg, *at_members(G, r, lane_node, members))
    # pause and unpause every group
    gids = np.arange(G, dtype=np.uint32)
    (rows_o, po), (rows_g, pg) = eo.pause_groups(gids), eg.pause_groups(gids)
    assert np.array_equal(po, pg) and po.sum() > G // 2
    assert rows_o.tobytes() == rows_g.tobytes()
    live = rows_o.reshape(-1)
    live = live[live["state"] != abi.ST_FREE]
    for e in (eo, eg):
        e.load_rows(live)
    same_state(eo, eg, G)
    for r in range(10, 13):
        same_round(eo, eg, *at_members(G, r, lane_node, members))
    c = same_state(eo, eg, G)
    assert c["decisions_made"] > 10 * G
    compare_logs(eo, eg, L)
    for e in (eo, eg):
        e.close()


@pytest.mark.parametrize("lane_nodes,seed", [([103, 100, 104, 101], 71), ([104, 102, 100, 103, 101], 72)])
def test_view_change_then_rounds(oracle_lib, cuda_lib, lane_nodes, seed):
    """elections through gpx_handle_prepare_replies (tests/p1b_cases.py) in a 4- or 5-lane engine, lanes in no member
    order, groups of 5: the installed coordinators' nodeSlotNumbers as recorded, then rounds on top of them"""
    R, G = 5, 300
    rng = np.random.default_rng(seed)
    eg, eo = make_engine(cuda_lib, R, G, lane_nodes), make_engine(oracle_lib, R, G, lane_nodes)
    L = len(lane_nodes)
    elected = 0
    for rnd in range(3):
        st = rng.bit_generator.state
        preconditions(eg, R, G, rng)
        rng.bit_generator.state = st
        preconditions(eo, R, G, rng)
        els, reps = random_elections(R, G, rng, False, lane_nodes)
        got, want = eg.handle_prepare_replies(els, reps), eo.handle_prepare_replies(els, reps)
        assert_same_out(got, want)
        elected += int((want["verdict"] == abi.EL_MAJORITY).sum())
        assert_same_rows(eg, eo, R, G, rnd)
        for r in range(2):
            reqs, pay = make_requests(np.arange(G), payload_len=3, seed=seed, round_no=4 * rnd + r, entry_lane=r % L,
                                      entry_node=lane_nodes[r % L])
            same_round(eo, eg, reqs, pay)
            assert_same_rows(eg, eo, R, G, (rnd, r))
    assert elected > G // 4
    assert eg.counters()["decisions_made"] > G


# ---- input rules -----------------------------------------------------------------------------------------------------

def test_input_rules_of_the_engine(cuda_lib):
    check_input_rules(cuda_lib)


def test_refused_call_leaves_no_member_set_behind(oracle_lib, cuda_lib):
    """a refused gpx_create_groups / gpx_load_rows whose first record introduced a member set, then a call that uses
    that set: the device must hold the set's lane mapping (a refused call once interned it on the host only)"""
    es = [small_engine(lib) for lib in (oracle_lib, cuda_lib)]
    for e in es:
        e.create_groups(descs([[100, 101, 102]] * 8))
        refused(abi.GPX_ERANGE, e.create_groups,
                np.concatenate([descs([[101, 100, 103]], gid0=8), descs([[100]], gid0=64)]))
        rows = e.dump_rows(np.arange(2), 0)
        rows["gid"] = [12, 13]
        rows["members"][0, :3] = [104, 100, 102]
        rows["lane"][1] = 3
        refused(abi.GPX_ERANGE, e.load_rows, rows)
        e.create_groups(descs([[101, 100, 103]] * 4 + [[104, 102, 100]] * 4, gid0=8))
    eo, eg = es
    same_state(eo, eg, 64)
    for r in range(4):
        reqs, pay = make_requests(np.arange(16), payload_len=4, seed=5, round_no=r, entry_lane=r % 3,
                                  entry_node=100 + r % 3)
        st, _ = same_round(eo, eg, reqs, pay)
    assert (st[8:] > 0).sum() >= 4, "groups with the new member sets decided"
    same_state(eo, eg, 64)
    compare_logs(eo, eg, 3)
    for e in es:
        e.close()


def test_member_set_limit(oracle_lib, cuda_lib):
    """the 4097th distinct member set is refused with its whole call; the engine keeps agreeing with the oracle"""
    eo, eg = mset_limit_engine(oracle_lib), mset_limit_engine(cuda_lib)
    G = MAX_MSETS + 1
    for r in range(3):
        reqs, pay = make_requests(np.arange(G), payload_len=2, seed=6, round_no=r, entry_lane=r % 2,
                                  entry_node=100 + r % 2)  # node 102 holds no instance of most groups
        st, _ = same_round(eo, eg, reqs, pay)
    assert (st > 0).sum() > G // 2 and (st == abi.RS_FORWARD).sum() > G // 8
    same_state(eo, eg, MAX_MSETS + 8)
    for e in (eo, eg):
        e.close()
