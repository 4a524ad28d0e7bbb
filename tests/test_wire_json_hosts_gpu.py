"""GPU: records decoded from JSON drive the engine as the byte forms' records do.

* Two hosts: engine A serves node 100, engine B nodes 101 and 102 (the scenario of tests/test_wire_device_gpu.py).  B's
  replies reach A, and A's commits reach B, only as JSON -- BatchedAcceptReply / BatchedCommit members written by
  packets_json's encoders, grouped into BATCHED_PAXOS_PACKET wrappers and bare packets -- decoded by
  gpx_wire_decode_json_device and handed to gpx_replies_device / gpx_decisions_device.  EXEC records, rows and counters
  equal one oracle engine.
* Preemption: a NACK from an acceptor that holds a higher ballot reaches the coordinator as a singleton JSON
  ACCEPT_REPLY (type 8).  Routed to the receiving node, not to the ballot's coordinator, it leaves the coordinator's
  state exactly as delivering the acceptor's reply record directly does -- destination the coordinator's member index,
  flag bits clear -- on the device and in the oracle.
* Lengths beyond the arena: GPX_EINVAL, nothing written.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import Engine, abi, make_config, make_requests
from test_wire_dev_gpu import accept_packets, by_node
from test_wire_device_gpu import DEV, DevNode, dev_recs, dptr, exec_and_extra
from wire_json_cases import group_into_packets

from gigapaxos_b200 import packets_json as pj, wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu


def json_arena(pkts, node):
    """(arena, refs) device tensors of JSON packets received by `node`"""
    arena, refs = wire.pack_packets(pkts)
    refs["node"] = node
    return (torch.from_numpy(arena.copy()).to(DEV),
            torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16).copy()).to(DEV))


def host_packets(enc: wire.EncodeOut, sel=None):
    out = enc.out.cpu().numpy()
    refs = wire.to_records(enc.refs, abi.wire_ref_dtype)
    if sel is not None:
        refs = refs[sel]
    return [bytes(out[int(r["off"]): int(r["off"]) + int(r["len"])]) for r in refs]


def replies_as_json(pkts):
    out = []
    for b in pkts:
        d = wire.decode_batched_accept_reply(b)
        out.append(pj.batched_accept_reply_json(d["paxos_id"], d["version"], d["acceptor"], d["bnum"], d["bcoord"],
                                                d["slot_number"], d["max_cp"], d["req_ids"][0] if d["req_ids"] else 0,
                                                d["slots"], d["req_ids"]))
    return out


def commits_as_json(pkts):
    out = []
    for b in pkts:
        d = wire.decode_batched_commit(b)
        out.append(pj.batched_commit_json(d["paxos_id"], d["version"], d["bnum"], d["bcoord"], d["median_cp"], d["slots"],
                                          d["group"]))
    return out


def group_setup(G, R):
    members = [100, 101, 102, 103, 104][:R]
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    descs = np.zeros(G, abi.group_desc_dtype)
    descs["gid"] = np.arange(G)
    descs["name_hash"] = [abi.java_string_hash(s) for s in names]
    descs["n_members"] = R
    descs["members"][:, :R] = members
    descs["init_mode"] = abi.INIT_BATCH
    coord = np.array([coordinator_of(s, members) for s in names])
    return members, names, descs, np.nonzero(coord == 100)[0]


def same_state(engines_lanes, gids):
    (e0, l0), rest = engines_lanes[0], engines_lanes[1:]
    r0 = e0.dump_rows(gids, l0)
    for e, l in rest:
        r = e.dump_rows(gids, l)
        for f in abi.row_dtype.names:
            if f != "lane":
                assert np.array_equal(r0[f], r[f]), f
    return r0


@pytest.mark.parametrize("R,window", [(3, 8), (5, 1)])
def test_two_hosts_over_json_wrappers_equal_one_oracle_engine(cuda_lib, oracle_lib, R, window):
    G = 512
    members, names, descs, gids = group_setup(G, R)
    common = dict(max_groups=G, window=window, max_group_size=R, max_batch_recs=4 * G)
    A = Engine(cuda_lib, make_config(cuda_lib, n_lanes=1, lane_node=[100], **common))
    B = Engine(cuda_lib, make_config(cuda_lib, n_lanes=2, lane_node=[101, 102], **common))
    O = Engine(oracle_lib, make_config(oracle_lib, n_lanes=3, lane_node=[100, 101, 102], **common))
    for e in (A, B, O):
        e.create_groups(descs)
    for e in (A, B):
        wire.set_group_names(e, gids, [names[g] for g in gids])
    dA, dB = DevNode(A), DevNode(B)
    rng = np.random.default_rng(R * 10 + window)
    got = {100: [], 101: [], 102: []}
    want = {100: [], 101: [], 102: []}
    rounds = 4
    for r in range(rounds):
        stop = np.zeros(len(gids), bool) if r < rounds - 1 else (gids % 7 == 0)
        reqs, pay = make_requests(gids, payload_len=5 + r, seed=3, round_no=r, entry_lane=0, entry_node=100,
                                  stop_mask=stop)
        acc_a, blob_a, st_a = A.propose(reqs, pay)
        acc_o, blob_o, st_o = O.propose(reqs, pay)
        assert np.array_equal(st_a, st_o) and (st_a > 0).all()
        # A -> B: ACCEPT bytes, as in the byte scenario
        arena, refs = wire.device_packets(accept_packets(names, 0, acc_a, blob_a))
        d = wire.decode_batch_device(B, arena, refs, (len(acc_a), 64 * len(acc_a), 1, 1))
        assert (d.status == abi.WS_OK).all()
        ctl_b, extra_b = dB.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_b = dB.accepts(d, ctl_b, extra_b)
        enc = wire.encode_replies_device(B, rep_b, rep_b.shape[0], (64 * len(acc_a), 2 * len(acc_a)))
        # B -> A: the replies only as JSON, in wrappers and bare
        pk = host_packets(enc)
        jpk, _ = group_into_packets(rng, replies_as_json(pk))
        ja, jr = json_arena(jpk, 100)
        j = wire.decode_json_device(A, ja, jr, (len(pk), 4 * len(acc_a), 1))
        assert (j.status == abi.WS_OK).all()
        assert (wire.to_records(j.members, abi.wire_member_dtype)["status"] == abi.WS_OK).all()
        byte_dec = wire.decode_batch_device(A, enc.out.clone(), enc.refs.clone(), (1, 16, 4 * len(acc_a), 1))
        assert torch.equal(j.replies, byte_dec.replies)  # the same records as the byte forms give
        rep_a, _ = A.handle_accepts(acc_a, blob_a)
        rep_o, _ = O.handle_accepts(acc_o, blob_o)
        ctl_a = dA.ctl()
        dec_a = torch.empty((4 * len(gids), 32), dtype=torch.uint8, device=DEV)
        dA.replies(dev_recs(rep_a, 32), len(rep_a), dec_a, ctl_a)
        dA.replies(j.replies, j.sizes[1], dec_a, ctl_a)
        dec_o = O.handle_accept_replies(rep_o)
        # A -> B: the commits only as JSON
        enc2 = wire.encode_decisions_device(A, dec_a, ctl_a.data_ptr() + 4, dec_a.shape[0], (64 * len(gids), 8 * len(gids)))
        n_dec = int(ctl_a[1].item())
        assert n_dec == len(dec_o) == len(gids)
        cpk = host_packets(enc2, wire.to_records(enc2.refs, abi.wire_ref_dtype)["node"] == 101)
        jpk2, _ = group_into_packets(rng, commits_as_json(cpk))
        ja2, jr2 = json_arena(jpk2, 101)
        j2 = wire.decode_json_device(B, ja2, jr2, (len(cpk), 1, 4 * len(gids)))
        assert (j2.status == abi.WS_OK).all() and j2.sizes[2] == len(gids)
        ctl_ax, extra_a = dA.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        ex_a = dA.decisions(dec_a, n_dec, extra_a, ctl_ax)
        ctl_bx = dB.ctl()
        extra_b.zero_()
        ex_b = dB.decisions(j2.decisions, j2.sizes[2], extra_b, ctl_bx)
        ex_o, x_o = O.handle_decisions(dec_o)
        for dct, ex in ((got, by_node(exec_and_extra(ex_a, extra_a, ctl_ax), [100])),
                        (got, by_node(exec_and_extra(ex_b, extra_b, ctl_bx), [101, 102])),
                        (want, by_node(np.concatenate([ex_o, x_o]), [100, 101, 102]))):
            for node, v in ex.items():
                dct[node].extend(v)
    for node in (100, 101, 102):
        assert got[node] == want[node] and len(want[node]) == rounds * len(gids)
    for eng, lane, olane in ((A, 0, 0), (B, 0, 1), (B, 1, 2)):
        same_state([(eng, lane), (O, olane)], gids)
    ca, cb, co = A.counters(), B.counters(), O.counters()
    for k in ("decisions_made", "executed", "stops_executed", "accepts_handled", "replies_handled"):
        assert ca[k] + cb[k] == co[k], k
    for e in (A, B, O):
        e.close()


def test_a_json_nack_preempts_the_coordinator_as_the_reply_record_does(cuda_lib, oracle_lib):
    """coordinator engines on node 100 only: A gets the remote replies as JSON (NACKs as type 8, positive replies as
    type 34), D (device) and O (oracle) get the same replies as records"""
    G = 300
    members, names, descs, gids = group_setup(G, 3)
    common = dict(max_groups=G, window=4, max_group_size=3, max_batch_recs=4 * G, n_lanes=1, lane_node=[100])
    A = Engine(cuda_lib, make_config(cuda_lib, **common))
    D = Engine(cuda_lib, make_config(cuda_lib, **common))
    O = Engine(oracle_lib, make_config(oracle_lib, **common))
    for e in (A, D, O):
        e.create_groups(descs)
    wire.set_group_names(A, gids, [names[g] for g in gids])
    reqs, pay = make_requests(gids, payload_len=7, seed=5, round_no=0, entry_lane=0, entry_node=100)
    props = [e.propose(reqs, pay) for e in (A, D, O)]
    assert all(np.array_equal(p[2], props[0][2]) for p in props)
    acc = props[0][0]
    own = [e.handle_accepts(p[0], p[1])[0] for e, p in zip((A, D, O), props)]
    before = O.dump_rows(gids, 0)
    recs = np.zeros(len(acc), abi.reply_dtype)
    pkts, nack = [], np.zeros(len(acc), bool)
    for i, a in enumerate(acc):
        gid, slot, bn, bc = int(a["gid"]), int(a["slot"]), int(a["bnum"]), int(a["bcoord"])
        rid = ((int(a["req_id"]) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)
        nack[i] = i % 3 == 0
        if nack[i]:  # acceptor 101 has promised its own higher ballot: its coordinator is 101, not the receiver
            recs[i] = (gid, slot, bn + 1, 101, slot - 1, abi.who(1, 0, 0), rid)
            pkts.append(pj.accept_reply_json(names[gid], 0, 101, bn + 1, 101, slot, slot - 1, rid))
        else:
            recs[i] = (gid, slot, bn, bc, slot - 1, abi.who(1, 0, 0), rid)
            pkts.append(pj.batched_accept_reply_json(names[gid], 0, 101, bn, bc, slot, slot - 1, rid, [slot], [rid]))
    bare = [p for p, n in zip(pkts, nack) if n]
    wrapped = [p for p, n in zip(pkts, nack) if not n]
    ja, jr = json_arena(bare + [pj.batched_paxos_packet_json(wrapped[k: k + 40]) for k in range(0, len(wrapped), 40)], 100)
    j = wire.decode_json_device(A, ja, jr, (len(pkts), len(pkts), 1))
    assert (j.status == abi.WS_OK).all()
    assert (wire.to_records(j.members, abi.wire_member_dtype)["status"] == abi.WS_OK).all()
    # the decoded replies are the records, regrouped by gid: bare NACKs first within a group, none shares one here
    assert np.array_equal(wire.to_records(j.replies, abi.reply_dtype), recs)
    dA = DevNode(A)
    ctl = dA.ctl()
    dec_a = torch.empty((4 * len(gids), 32), dtype=torch.uint8, device=DEV)
    dA.replies(dev_recs(own[0], 32), len(own[0]), dec_a, ctl)
    dA.replies(j.replies, j.sizes[1], dec_a, ctl)
    got = wire.to_records(dec_a[: int(ctl[1].item())], abi.decision_dtype)
    outs = []
    for e, rep in ((D, own[1]), (O, own[2])):
        outs.append(np.concatenate([e.handle_accept_replies(rep), e.handle_accept_replies(recs)]))
    assert np.array_equal(got, outs[0]) and np.array_equal(got, outs[1])
    assert len(got) == int((~nack).sum())  # every positive reply makes a majority with the coordinator's own
    after = same_state([(A, 0), (D, 0), (O, 0)], gids)
    # the NACKs preempted their coordinators: the groups' coordinator state moved, the others' did not
    moved = (after["coord_active"] != before["coord_active"]) | (after["coord_bnum"] != before["coord_bnum"]) | \
        (after["coord_bcoord"] != before["coord_bcoord"]) | (after["coord_exists"] != before["coord_exists"])
    pos = {int(g): i for i, g in enumerate(gids)}
    idx = np.array([pos[int(a["gid"])] for a in acc])
    assert moved[idx[nack]].all() and not moved[idx[~nack]].any()
    ca, cd, co = A.counters(), D.counters(), O.counters()
    for k in ("decisions_made", "replies_handled", "accepts_handled"):
        assert ca[k] == cd[k] == co[k], k
    for e in (A, D, O):
        e.close()


def test_lengths_beyond_the_arena_are_refused(cuda_lib):
    G = 8
    members, names, descs, gids = group_setup(G, 3)
    A = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, max_group_size=3, n_lanes=1, lane_node=[100]))
    A.create_groups(descs)
    wire.set_group_names(A, gids, [names[g] for g in gids])
    pk = pj.batched_commit_json(names[int(gids[0])], 0, 1, 100, 0, list(range(300)), members)  # many chunks long
    arena, refs = wire.pack_packets([pk])
    many = np.repeat(refs, 64)
    da = torch.from_numpy(arena.copy()).to(DEV)
    dr = torch.from_numpy(many.view(np.uint8).reshape(len(many), 16).copy()).to(DEV)
    bufs = [torch.full((1 << 12,), 0xAB, dtype=torch.uint8, device=DEV) for _ in range(3)]
    status = torch.zeros(len(many), dtype=torch.int32, device=DEV)
    sz = [C.c_uint32(64) for _ in range(3)]
    rc = A.L.fn("wire_decode_json_device")(A.handle, C.c_uint32(len(many)), dptr(da), C.c_uint64(da.numel()), dptr(dr),
                                           dptr(status), dptr(bufs[0]), C.byref(sz[0]), dptr(bufs[1]), C.byref(sz[1]),
                                           dptr(bufs[2]), C.byref(sz[2]), wire.stream_handle())
    assert rc == abi.GPX_EINVAL
    torch.cuda.synchronize()
    assert all(bool((b == 0xAB).all()) for b in bufs)
    A.close()
