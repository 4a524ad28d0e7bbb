"""GPU: gpx_wire_encode_json_device through the C ABI.

* Bytes: random worlds with hard names, 1-8 lanes, unnamed groups and a device decision count give exactly the output
  of the Python model (tests/wire_json_out_cases.py); at 100 K groups the wrappers are cut at the real 4 MiB.
* Two hosts: engine A (node 100) and engine B (nodes 101, 102) exchange the JSON form -- B's replies and A's commits as
  BATCHED_PAXOS_PACKET wrappers, decoded with gpx_wire_decode_json_device -- and end with the EXEC records and rows of
  the same chain run with the byte encoders and decoder, at 512 and at 100 K groups.
"""
import numpy as np
import pytest
import torch

from helpers import Engine, abi, make_config, make_requests
from test_wire_dev_gpu import accept_packets, by_node
from test_wire_device_gpu import DevNode, dev_recs, exec_and_extra, ref_nodes
from wire_json_out_cases import expected_json, json_decisions, json_replies, json_world

from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu

NODES = [100, 101, 102, 98, 99, 97, 96, 95]


def engine_of(cuda_lib, world, named, **kw):
    G = max(world.groups) + 1
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, max_group_size=16, n_lanes=len(world.lanes),
                                     lane_node=world.lanes, **kw))
    d = np.zeros(G, abi.group_desc_dtype)
    for gid, (name, ver, members) in world.groups.items():
        d[gid] = (gid, ver, abi.java_string_hash(name), len(members), list(members) + [0] * (16 - len(members)),
                  abi.INIT_BATCH)
    e.create_groups(d)
    named = sorted(named)
    wire.set_group_names(e, named, [world.groups[g][0] for g in named])
    return e


def run(e, rep, dec, n_dec=None, wrap=0, caps=(1, 1)):
    drep = dev_recs(rep, 32) if len(rep) else None
    ddec = dev_recs(dec, 32) if len(dec) else None
    cnt = torch.tensor([n_dec], dtype=torch.int32, device="cuda") if n_dec is not None else None
    o = wire.encode_json_device(e, drep, len(rep), ddec, cnt.data_ptr() if cnt is not None else None, len(dec), caps,
                                wrap)
    refs = wire.to_records(o.refs, abi.wire_ref_dtype)
    return (o.rstatus_replies.cpu().numpy(), o.rstatus_decisions.cpu().numpy(), o.out.cpu().numpy().tobytes(),
            [(int(r["off"]), int(r["len"]), int(r["gid"]), int(r["node"])) for r in refs])


@pytest.mark.parametrize("lanes", [1, 3, 8])
def test_output_equals_the_model(cuda_lib, lanes):
    rng = np.random.default_rng(lanes)
    world = json_world(rng, 60, NODES[:lanes], permute=False)
    named = set(world.groups) - {0, 1}
    e = engine_of(cuda_lib, world, named)
    rep, dec = json_replies(rng, world, 300, lanes), json_decisions(rng, world, 400)
    for n_dec, wrap in ((None, 0), (250, abi.GPX_JSON_MAX_MEMBER + 3000)):
        rr, rd, out, refs = run(e, rep, dec, n_dec, wrap)
        er, ed, eout, erefs = expected_json(world, named, rep, dec, n_dec, wrap or abi.GPX_JSON_WRAP_BYTES)
        assert list(rr) == list(er) and list(rd[: len(ed)]) == list(ed)
        assert out == eout and refs == erefs and len(refs) > 10
    e.close()


def test_wrappers_are_cut_at_4_mib_at_100k_groups(cuda_lib):
    rng = np.random.default_rng(5)
    G = 100_000
    groups = {g: (f"grp/{g}é\"", 0, [100, 103]) for g in range(G)}
    from wire_dev_cases import World
    world = World(groups, [100])
    e = engine_of(cuda_lib, world, set(groups))
    rep = np.zeros(G, abi.reply_dtype)
    rep["gid"], rep["slot"], rep["bnum"], rep["bcoord"] = np.arange(G), (1 << 31) - 1, 7, 103
    rep["who"], rep["req_id"] = abi.who(0, 1, 0), rng.integers(-(1 << 62), 1 << 62, G)
    dec = np.zeros(G, abi.decision_dtype)
    dec["gid"], dec["slot"], dec["bnum"], dec["bcoord"], dec["flags"] = np.arange(G), 5, 7, 100, abi.F_DECISION
    rr, rd, out, refs = run(e, rep, dec)
    er, ed, eout, erefs = expected_json(world, set(groups), rep, dec)
    assert out == eout and refs == erefs
    assert len(refs) >= 3 and max(n for _, n, _, _ in refs) <= abi.GPX_JSON_WRAP_BYTES
    assert max(n for _, n, _, _ in refs) > abi.GPX_JSON_WRAP_BYTES - 2 * abi.GPX_JSON_MAX_MEMBER
    e.close()


def chain(cuda_lib, G, json_form):
    """A (node 100) coordinates, B (nodes 101, 102) accepts; -> (EXEC by engine, rows by (engine, lane))"""
    R, members = 3, [100, 101, 102]
    names = [f"NoopPaxosApp{g}ÿ" for g in range(G)]
    descs = np.zeros(G, abi.group_desc_dtype)
    descs["gid"] = np.arange(G)
    descs["name_hash"] = [abi.java_string_hash(s) for s in names]
    descs["n_members"] = R
    descs["members"][:, :R] = members
    descs["init_mode"] = abi.INIT_BATCH
    coord = np.array([coordinator_of(s, members) for s in names])
    gids = np.nonzero(coord == 100)[0]
    common = dict(max_groups=G, window=8, max_group_size=R, max_batch_recs=4 * G)
    A = Engine(cuda_lib, make_config(cuda_lib, n_lanes=1, lane_node=[100], **common))
    B = Engine(cuda_lib, make_config(cuda_lib, n_lanes=2, lane_node=[101, 102], **common))
    for e in (A, B):
        e.create_groups(descs)
        wire.set_group_names(e, gids, [names[g] for g in gids])
    dA, dB = DevNode(A), DevNode(B)
    ex = {"A": [], "B": []}
    for r in range(3):
        reqs, pay = make_requests(gids, payload_len=5 + r, seed=3, round_no=r, entry_lane=0, entry_node=100)
        acc_a, blob_a, st_a = A.propose(reqs, pay)
        assert (st_a > 0).all()
        arena, refs = wire.device_packets(accept_packets(names, 0, acc_a, blob_a))
        d = wire.decode_batch_device(B, arena, refs, (1, 16, 1, 1))
        ctl_b, extra_b = dB.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device="cuda")
        rep_b = dB.accepts(d, ctl_b, extra_b)
        rep_a, _ = A.handle_accepts(acc_a, blob_a)
        ctl_a = dA.ctl()
        dec_a = torch.empty((4 * len(gids), 32), dtype=torch.uint8, device="cuda")
        dA.replies(dev_recs(rep_a, 32), len(rep_a), dec_a, ctl_a)
        if json_form:  # B -> A: reply wrappers; A -> B: commit wrappers, each decoded as JSON
            enc = wire.encode_json_device(B, rep_b, rep_b.shape[0], None, None, 0, (64, 1))
            assert (ref_nodes(enc.refs) == 100).all()
            d2 = wire.decode_json_device(A, enc.out.clone(), enc.refs.clone(), (1, 1, 1))
            assert (d2.status == abi.WS_OK).all()
            dA.replies(d2.replies, d2.sizes[1], dec_a, ctl_a)
            enc2 = wire.encode_json_device(A, None, 0, dec_a, ctl_a.data_ptr() + 4, dec_a.shape[0], (64, 1))
            sel = ref_nodes(enc2.refs) == 101
            d3 = wire.decode_json_device(B, enc2.out.clone(), enc2.refs[sel].contiguous(), (1, 1, 1))
            assert (d3.status == abi.WS_OK).all()
            bdec, n_bdec = d3.decisions, d3.sizes[2]
        else:
            enc = wire.encode_replies_device(B, rep_b, rep_b.shape[0], (64, 1))
            d2 = wire.decode_batch_device(A, enc.out.clone(), enc.refs.clone(), (1, 16, 1, 1))
            dA.replies(d2.replies, d2.sizes[2], dec_a, ctl_a)
            enc2 = wire.encode_decisions_device(A, dec_a, ctl_a.data_ptr() + 4, dec_a.shape[0], (64, 1))
            sel = ref_nodes(enc2.refs) == 101
            d3 = wire.decode_batch_device(B, enc2.out.clone(), enc2.refs[sel].contiguous(), (1, 16, 1, 1))
            bdec, n_bdec = d3.decisions, d3.sizes[3]
        n_dec = int(ctl_a[1].item())
        assert n_dec == len(gids) and n_bdec == len(gids)
        ctl_ax, extra_a = dA.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device="cuda")
        ex_a = dA.decisions(dec_a, n_dec, extra_a, ctl_ax)
        ctl_bx = dB.ctl()
        extra_b.zero_()
        ex_b = dB.decisions(bdec, n_bdec, extra_b, ctl_bx)
        # per node, in (gid, slot) order: the tally's decisions, and so the EXEC records, come in no fixed order
        ex["A"].append(by_node(exec_and_extra(ex_a, extra_a, ctl_ax), [100]))
        ex["B"].append(by_node(exec_and_extra(ex_b, extra_b, ctl_bx), [101, 102]))
    rows = {(k, lane): eng.dump_rows(gids, lane).tobytes() for k, eng, lanes in (("A", A, 1), ("B", B, 2))
            for lane in range(lanes)}
    for e in (A, B):
        e.close()
    return ex, rows


@pytest.mark.parametrize("G", [512, 100_000])
def test_two_hosts_over_json_equal_the_byte_chain(cuda_lib, G):
    ex_j, rows_j = chain(cuda_lib, G, True)
    ex_b, rows_b = chain(cuda_lib, G, False)
    assert ex_j == ex_b and all(len(x[100]) == len(ex_b["A"][0][100]) > 0 for x in ex_b["A"])
    assert rows_j == rows_b
