"""GPU: the phase-2 wire calls through the C ABI (gpx_set_group_names, gpx_wire_decode_batch, gpx_wire_encode_*).

* Bytes: the cases of tests/test_wire_dev.py on the device, against the host codec (tests/wire_dev_cases.py).
* Two hosts: engine A serves node 100, engine B nodes 101 and 102, as two machines would.  ACCEPTs that A proposes are
  encoded by the host codec and decoded by B on the device; B's replies are encoded and decoded on the device back at
  A; A's decisions likewise at B.  The EXEC records and rows of every node must equal those of ONE oracle engine that
  hosts all three nodes as lanes (the method of test_spread_c_gpu.py).
* Scale: the name table at 1 M gids through set, lookup, destroy, re-create at version + 1 and pause.
"""
import numpy as np
import pytest

from helpers import Engine, abi, group_descs_fast, java_hash_numbered, make_config, make_requests
from wire_dev_cases import (World, check_decode, expected_encode_decisions, expected_encode_replies, malformed_packets,
                            random_decisions, random_packets, random_replies, random_world)

from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu


def world_engine(cuda_lib, world: World, **kw):
    G = max(world.groups) + 1
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, max_group_size=16, n_lanes=len(world.lanes),
                                     lane_node=world.lanes, **kw))
    d = np.zeros(G, abi.group_desc_dtype)
    for gid, (name, ver, members) in world.groups.items():
        d[gid] = (gid, ver, abi.java_string_hash(name), len(members), list(members) + [0] * (16 - len(members)),
                  abi.INIT_BATCH)
    e.create_groups(d)
    wire.set_group_names(e, list(world.groups), [g[0] for g in world.groups.values()])
    return e


@pytest.mark.parametrize("seed", [1, 2])
def test_device_decode_and_encode_match_the_host_codec(cuda_lib, seed):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 60)
    e = world_engine(cuda_lib, world)
    pkts, srcs = random_packets(rng, world, 2000)
    check_decode(world, pkts, srcs, wire.decode_batch(e, pkts))
    cases = malformed_packets(world)
    st = wire.decode_batch(e, [p for p, _ in cases])[0]
    assert list(st) == [s for _, s in cases]
    L = len(world.lanes)
    rep = random_replies(rng, world, 500, L)
    rst, arena, refs = wire.encode_replies(e, rep)
    est, exp = expected_encode_replies(world, rep, L)
    assert np.array_equal(rst, est) and wire.unpack_packets(arena, refs) == exp
    dec = random_decisions(rng, world, 800)
    rst, arena, refs = wire.encode_decisions(e, dec)
    est, exp = expected_encode_decisions(world, dec)
    assert np.array_equal(rst, est) and wire.unpack_packets(arena, refs) == exp
    e.close()


def test_a_name_is_refused_while_another_live_gid_holds_it(cuda_lib):
    world = random_world(np.random.default_rng(3), 4)
    e = world_engine(cuda_lib, world)
    with pytest.raises(abi.GpxError):
        wire.set_group_names(e, [1], [world.groups[0][0]])
    with pytest.raises(abi.GpxError):
        wire.set_group_names(e, [1, 2], ["x", "x"])
    wire.set_group_names(e, [0, 1], [world.groups[1][0], world.groups[0][0]])  # a swap inside one call is fine
    e.close()


def exec_key(ex):
    ok = (ex["flags"] & abi.F_VOID) == 0
    x = ex[ok]
    lanes = (x["flags"] >> 12) & 0xF
    return lanes, x


def by_node(ex, lanes_nodes):
    lanes, x = exec_key(ex)
    out = {}
    for l, node in enumerate(lanes_nodes):
        y = x[lanes == l]
        y = y[np.lexsort((y["slot"], y["gid"]))]
        out[node] = [(int(a["gid"]), int(a["slot"]), int(a["req_id"]), int(a["flags"]) & ~(0xF << 12)) for a in y]
    return out


def accept_packets(names, version, accepts, blob):
    pk = []
    for a in accepts:
        val = bytes(blob[int(a["payload_off"]): int(a["payload_off"]) + int(a["payload_len"])])
        assert int(a["nreq"]) == 1
        req = wire.Request(names[int(a["gid"])], version, int(a["req_id"]), val, stop=bool(a["flags"] & abi.F_STOP),
                           entry_replica=100, entry_time=0)
        pk.append(wire.encode_accept(req, int(a["slot"]), int(a["bnum"]), int(a["bcoord"]), False, int(a["median_cp"]),
                                     int(a["sender"])))
    return pk


def merge_by_gid(*arrs):
    x = np.concatenate([a for a in arrs if len(a)]) if any(len(a) for a in arrs) else arrs[0][:0]
    return x[np.argsort(x["gid"], kind="stable")]


@pytest.mark.parametrize("R,window", [(3, 8), (5, 1), (3, 1), (5, 8)])
def test_two_hosts_over_device_wire_equal_one_oracle_engine(cuda_lib, oracle_lib, R, window):
    G = 512
    members = [100, 101, 102, 103, 104][:R]
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    descs = np.zeros(G, abi.group_desc_dtype)
    descs["gid"] = np.arange(G)
    descs["name_hash"] = [abi.java_string_hash(s) for s in names]
    descs["n_members"] = R
    descs["members"][:, :R] = members
    descs["init_mode"] = abi.INIT_BATCH
    coord = np.array([coordinator_of(s, members) for s in names])
    gids = np.nonzero(coord == 100)[0]  # groups that node 100 coordinates
    common = dict(max_groups=G, window=window, max_group_size=R, max_batch_recs=4 * G)
    A = Engine(cuda_lib, make_config(cuda_lib, n_lanes=1, lane_node=[100], **common))
    B = Engine(cuda_lib, make_config(cuda_lib, n_lanes=2, lane_node=[101, 102], **common))
    O = Engine(oracle_lib, make_config(oracle_lib, n_lanes=3, lane_node=[100, 101, 102], **common))
    for e in (A, B, O):
        e.create_groups(descs)
    for e in (A, B):
        wire.set_group_names(e, gids, [names[g] for g in gids])
    got = {100: [], 101: [], 102: []}
    want = {100: [], 101: [], 102: []}
    rounds = 5
    for r in range(rounds):
        stop = np.zeros(len(gids), bool) if r < rounds - 1 else (gids % 7 == 0)
        reqs, pay = make_requests(gids, payload_len=5 + r, seed=3, round_no=r, entry_lane=0, entry_node=100,
                                  stop_mask=stop)
        acc_a, blob_a, st_a = A.propose(reqs, pay)
        acc_o, blob_o, st_o = O.propose(reqs, pay)
        assert np.array_equal(st_a, st_o) and (st_a > 0).all()
        # A -> B: ACCEPTs as bytes, plus one for a group B has no name for
        pk = accept_packets(names, 0, acc_a, blob_a)
        unnamed = wire.encode_batched_commit("NoSuchGroup", 0, 0, 100, 0, [1], members)
        status, acc_b, blob_b, rep_x, dec_x = wire.decode_batch(B, pk + [unnamed])
        assert (status[:-1] == abi.WS_OK).all() and status[-1] == abi.WS_UNKNOWN_NAME
        assert len(rep_x) == len(dec_x) == 0 and len(acc_b) == len(acc_a)
        rep_a, _ = A.handle_accepts(acc_a, blob_a)
        rep_b, _ = B.handle_accepts(acc_b, blob_b)
        rep_o, _ = O.handle_accepts(acc_o, blob_o)
        # B -> A: replies encoded and decoded on the device
        rst, arena, refs = wire.encode_replies(B, rep_b)
        assert (rst != abi.WE_NACK).all() and (refs["node"] == 100).all()
        st, _, _, rep_ab, _ = wire.decode_batch(A, [p for _, _, p in wire.unpack_packets(arena, refs)])
        assert (st == abi.WS_OK).all()
        dec_a = A.handle_accept_replies(merge_by_gid(rep_a, rep_ab))
        dec_o = O.handle_accept_replies(rep_o)
        assert len(dec_a) == len(dec_o) == len(gids)
        # A -> B: decisions encoded and decoded on the device (one commit, indexed for 101 and 102 and any absent node)
        rst, arena, refs = wire.encode_decisions(A, dec_a)
        assert (rst == abi.WE_SENT).all() and len(refs) == len(gids) * (R - 1)
        pk = {}
        for gid, node, p in wire.unpack_packets(arena, refs):
            if node == 101:
                pk[gid] = p
        st, _, _, _, dec_b = wire.decode_batch(B, [pk[g] for g in sorted(pk)])
        assert (st == abi.WS_OK).all()
        ex_a, x_a = A.handle_decisions(dec_a)
        ex_b, x_b = B.handle_decisions(dec_b)
        ex_o, x_o = O.handle_decisions(dec_o)
        for d, ex in ((got, by_node(np.concatenate([ex_a, x_a]), [100])),
                      (got, by_node(np.concatenate([ex_b, x_b]), [101, 102])),
                      (want, by_node(np.concatenate([ex_o, x_o]), [100, 101, 102]))):
            for node, v in ex.items():
                d[node].extend(v)
    for node in (100, 101, 102):
        assert got[node] == want[node] and len(want[node]) == rounds * len(gids)
    for eng, lane, olane in ((A, 0, 0), (B, 0, 1), (B, 1, 2)):
        ra, ro = eng.dump_rows(gids, lane), O.dump_rows(gids, olane)
        for f in abi.row_dtype.names:
            if f != "lane":
                assert np.array_equal(ra[f], ro[f]), f
    ca, cb, co = A.counters(), B.counters(), O.counters()
    for k in ("decisions_made", "executed", "stops_executed", "accepts_handled", "replies_handled"):
        assert ca[k] + cb[k] == co[k], k
    for e in (A, B, O):
        e.close()


def test_two_hosts_a_bumped_ballot_is_a_nack_left_to_the_host(cuda_lib):
    name = next(f"grp{i}" for i in range(100) if coordinator_of(f"grp{i}", [100, 101, 102]) == 100)
    world = World({0: (name, 0, [100, 101, 102])}, lanes=[101, 102])
    B = world_engine(cuda_lib, world)  # the acceptors start at ballot (0, 100): node 100 coordinates
    req = wire.Request(name, 0, 9, b"v", entry_replica=100)
    p = wire.encode_accept(req, 0, 0, 100, False, -1, 100)
    _, acc, blob, _, _ = wire.decode_batch(B, [p])
    rep, _ = B.handle_accepts(acc, blob)
    patch = np.zeros(2, abi.patch_dtype)
    patch["gid"], patch["lane"], patch["op"], patch["a"], patch["b"] = 0, [0, 1], abi.PATCH_SET_BALLOT, 5, 101
    B.patch(patch)
    p2 = wire.encode_accept(wire.Request(name, 0, 10, b"w", entry_replica=100), 1, 0, 100, False, -1, 100)
    _, acc2, blob2, _, _ = wire.decode_batch(B, [p2])
    rep2, _ = B.handle_accepts(acc2, blob2)
    assert (abi.who_flags(rep2["who"]) & abi.F_NACK).all()
    rst, arena, refs = wire.encode_replies(B, np.concatenate([rep, rep2]))
    assert rst.tolist() == [abi.WE_SENT, abi.WE_SENT, abi.WE_NACK, abi.WE_NACK] and len(refs) == 2
    B.close()


def test_name_table_at_one_million_gids(cuda_lib):
    G = 1 << 20
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=3, window=1, max_batch_recs=1 << 16,
                                     log_ring_bytes=1 << 20))
    d = group_descs_fast(G)
    e.create_groups(d)
    gids = np.arange(G, dtype=np.uint32)
    names = [f"NoopPaxosApp{i}" for i in range(G)]
    wire.set_group_names(e, gids, names)
    sample = np.random.default_rng(5).choice(G, size=20000, replace=False)
    pk = [wire.encode_batched_commit(names[g], 0, 0, 100, 0, [1], [100, 101, 102]) for g in sample]
    st, _, _, _, dec = wire.decode_batch(e, pk)
    assert (st == abi.WS_OK).all() and sorted(dec["gid"].tolist()) == sorted(sample.tolist())
    # destroy a quarter, re-create it at version 1, pause another quarter
    q = gids[: G // 4]
    e.destroy_groups(q)
    st = wire.decode_batch(e, pk)[0]
    assert ((st == abi.WS_UNKNOWN_NAME) == (sample < G // 4)).all()
    d1 = d[: G // 4].copy()
    d1["version"] = 1
    e.create_groups(d1)
    wire.set_group_names(e, q, names[: G // 4])
    st = wire.decode_batch(e, pk)[0]
    assert ((st == abi.WS_VERSION) == (sample < G // 4)).all()
    _, paused = e.pause_groups(gids[G // 4: G // 2])
    assert paused.all()
    st = wire.decode_batch(e, pk)[0]
    assert ((st == abi.WS_UNKNOWN_NAME) == ((sample >= G // 4) & (sample < G // 2))).all()
    assert ((st == abi.WS_OK) == (sample >= G // 2)).all()
    # the freed names can be given to other gids, and every cell reused or rebuilt keeps lookups right
    wire.set_group_names(e, gids[G // 2: G // 2 + 1000], [f"renamed{i}" for i in range(1000)])
    pk2 = [wire.encode_batched_commit(f"renamed{i}", 0, 0, 100, 0, [1], [100, 101, 102]) for i in range(1000)]
    st, _, _, _, dec = wire.decode_batch(e, pk2)
    assert (st == abi.WS_OK).all() and dec["gid"].tolist() == list(range(G // 2, G // 2 + 1000))
    e.close()
