"""GPU: gpx_wire_encode_json_sweep_device through the C ABI.

* Bytes: random worlds with hard names, 1, 3 and 8 lanes, forwards entering at random lanes of a real engine (its
  routing rows read back with gpx_dump_rows) give exactly the output of the Python model
  (tests/wire_json_sweep_cases.py); rstatus_reqs is gpx_wire_encode_forwards_device's; with no requests every output is
  gpx_wire_encode_json_device's.  At 100 K groups the wrappers, forwards among replies, are cut at the real 4 MiB.
* Three nodes, as in test_wire_forward_gpu.py: client REQUEST packets enter at node 101's engine B for groups node 100
  (engine A) coordinates.  B sends each round's replies to A together with the next round's forwards, in one sweep; A
  takes replies and requests out of it with gpx_wire_decode_json_device, gpx_wire_decode_json_requests_device and, for
  the lone REQUEST packets, gpx_wire_decode_requests_device.  EXEC records and rows equal one oracle engine hosting
  all three nodes, at 512 and at 100 K groups.
"""
import numpy as np
import pytest
import torch

from helpers import Engine, abi, make_config, make_requests
from test_wire_coord_gpu import request_arena
from test_wire_dev_gpu import by_node
from test_wire_device_gpu import DevNode, dev_recs, exec_and_extra, host_bytes, ref_nodes
from test_wire_forward_gpu import engine_rows
from test_wire_json_out_gpu import NODES, engine_of, run as run_json
from wire_coord_cases import NOW_MS
from wire_dev_cases import World
from wire_json_out_cases import json_decisions, json_replies, json_world
from wire_json_sweep_cases import expected_sweep

from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu

DEV = "cuda"


def sweep(e, rep, dec, fwd_dev, n_dec=None, wrap=0, caps=(1, 1)):
    """fwd_dev = (reqs, meta, n, status, payload, down) on the device, or None"""
    drep = dev_recs(rep, 32) if rep is not None and len(rep) else None
    ddec = dev_recs(dec, 32) if dec is not None and len(dec) else None
    nr, nd = (len(rep) if rep is not None else 0), (len(dec) if dec is not None else 0)
    cnt = torch.tensor([n_dec], dtype=torch.int32, device=DEV) if n_dec is not None else None
    rq, mt, n, st, pay, down = fwd_dev if fwd_dev is not None else (None, None, 0, None, None, [])
    o = wire.encode_json_sweep_device(e, drep, nr, ddec, cnt.data_ptr() if cnt is not None else None, nd, rq, mt, n,
                                      st, pay, down, caps, wrap)
    refs = wire.to_records(o.refs, abi.wire_ref_dtype)
    return (o.rstatus_replies.cpu().numpy(), o.rstatus_decisions.cpu().numpy(), o.rstatus_reqs.cpu().numpy(),
            o.out.cpu().numpy().tobytes(), [(int(r["off"]), int(r["len"]), int(r["gid"]), int(r["node"])) for r in refs])


def proposed_forwards(e, world, rng, per_max=3, edge=True):
    """requests for every group, entering at a random lane per group, proposed on the device: (host (reqs, meta,
    status, payload), device (reqs, meta, n, status, payload))"""
    gids = np.array(sorted(world.groups), np.uint32)
    per = rng.integers(1, per_max + 1, size=len(gids))
    rg = np.repeat(gids, per)
    lane_of = rng.integers(0, len(world.lanes), size=int(gids.max()) + 1)
    reqs, pay = make_requests(rg, payload_len=rng.integers(0, 40, size=len(rg)), seed=int(rng.integers(1 << 20)))
    pay = pay.copy()
    pay[: len(pay) // 2] = rng.integers(0, 256, size=len(pay) // 2)  # quotes, backslashes, control bytes, >= 0x80
    reqs["flags"] = (reqs["flags"] & ~np.uint32(0xF00)) | (lane_of[rg].astype(np.uint32) << 8)
    meta = np.zeros(len(reqs), abi.req_meta_dtype)
    meta["client_ip"] = [10, 1, 2, 3]
    meta["client_port"] = rng.choice([0, 4567, 65535], size=len(reqs))
    meta["client_ip"][meta["client_port"] == 0] = 0
    meta["listen_ip"] = [1, 2, 3, 4]
    meta["listen_port"] = rng.choice([0, 80], size=len(reqs))
    meta["listen_ip"][meta["listen_port"] == 0] = 0
    meta["forward_count"] = rng.choice([0, 0, 1, 3, -1, (1 << 31) - 1] if edge else [0], size=len(reqs))
    meta["entry_time"] = rng.choice([0, 1 << 41, -(1 << 63), (1 << 63) - 1] if edge else [5], size=len(reqs))
    meta["flags"] = rng.choice([0, abi.RM_RETURN_VALUE, abi.RM_BROADCASTED], size=len(reqs))
    if edge:
        reqs["req_id"][::5] = rng.choice([-(1 << 63), (1 << 63) - 1, -1], size=len(reqs[::5]))
    n = len(reqs)
    d_reqs, d_meta, d_pay = dev_recs(reqs, 32), dev_recs(meta, 32), torch.from_numpy(pay).to(DEV)
    st = torch.empty(n, dtype=torch.int32, device=DEV)
    wire.propose_device_heads(e, d_reqs, n, d_pay, len(pay), st, torch.empty((n, 48), dtype=torch.uint8, device=DEV),
                              torch.empty(n, dtype=torch.int32, device=DEV),
                              torch.zeros(8, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    return (reqs, meta, st.cpu().numpy(), pay), (d_reqs, d_meta, n, st, d_pay)


@pytest.mark.parametrize("lanes", [1, 3, 8])
def test_output_equals_the_model_and_the_forwards_encoder(cuda_lib, lanes):
    rng = np.random.default_rng(20 + lanes)
    world = json_world(rng, 300, NODES[:lanes], permute=False)
    named = set(world.groups) - set(range(0, 300, 11))
    G = max(world.groups) + 1
    e = engine_of(cuda_lib, world, named, window=8, max_batch_recs=4 * G, max_batch_payload=64 * G)
    (reqs, meta, status, pay), (d_reqs, d_meta, n, st, d_pay) = proposed_forwards(e, world, rng)
    rows = engine_rows(e, np.arange(G, dtype=np.uint32), G, e.cfg)
    rep, dec = json_replies(rng, world, 200, lanes), json_decisions(rng, world, 300)
    for down, wrap in (([103], 0), ([], abi.GPX_JSON_MAX_MEMBER + 3000)):
        rr, rd, rq, out, refs = sweep(e, rep, dec, (d_reqs, d_meta, n, st, d_pay, down), wrap=wrap)
        er, ed, eq, eout, erefs, lone = expected_sweep(world, named, rep, dec, (rows, reqs, meta, status, pay, down),
                                                       wrap_bytes=wrap or abi.GPX_JSON_WRAP_BYTES)
        assert list(rr) == list(er) and list(rd) == list(ed) and list(rq) == list(eq)
        assert out == eout and refs == erefs and len(lone) > 0
        fw = wire.encode_forwards_device(e, d_reqs, d_meta, n, st, d_pay, down, (1, 1))
        assert host_bytes(fw.rstatus) == rq.tobytes()
        assert {abi.WE_SENT, abi.WE_VOID, abi.WE_NO_NAME} <= set(rq.tolist())
    # no requests: gpx_wire_encode_json_device's outputs
    for n_dec, wrap in ((None, 0), (120, abi.GPX_JSON_MAX_MEMBER + 1000)):
        a = sweep(e, rep, dec, None, n_dec, wrap)
        b = run_json(e, rep, dec, n_dec, wrap)
        assert a[0].tolist() == b[0].tolist() and a[1].tolist() == b[1].tolist() and a[2].size == 0
        assert a[3] == b[2] and a[4] == b[3]
    e.close()


def test_wrappers_with_forwards_are_cut_at_4_mib_at_100k_groups(cuda_lib):
    rng = np.random.default_rng(6)
    G = 100_000
    groups = {g: (f"grp/{g}é\"", 0, [100, 103]) for g in range(G)}
    world = World(groups, [100])
    e = engine_of(cuda_lib, world, set(groups), max_batch_recs=2 * G, max_batch_payload=64 * G)
    (reqs, meta, status, pay), fwd_dev = proposed_forwards(e, world, rng, per_max=1, edge=False)
    rows = engine_rows(e, np.arange(G, dtype=np.uint32), G, e.cfg)
    assert (status == abi.RS_FORWARD).sum() > G // 3
    rep = np.zeros(G, abi.reply_dtype)
    rep["gid"], rep["slot"], rep["bnum"], rep["bcoord"] = np.arange(G), (1 << 31) - 1, 7, 103
    rep["who"], rep["req_id"] = abi.who(0, 1, 0), rng.integers(-(1 << 62), 1 << 62, G)
    rr, rd, rq, out, refs = sweep(e, rep, None, fwd_dev + ([],))
    er, _, eq, eout, erefs, lone = expected_sweep(world, set(groups), rep, None, (rows, reqs, meta, status, pay, []))
    assert list(rq) == list(eq) and out == eout and refs == erefs and lone == []
    sizes = [n for _, n, _, _ in refs]
    assert len(refs) > 3 and max(sizes) <= abi.GPX_JSON_WRAP_BYTES and max(sizes) > abi.GPX_JSON_WRAP_BYTES - (1 << 17)
    e.close()


# ---- three nodes: a round's replies and the next round's forwards in one sweep ------------------------------------------
def repack(parts):
    """request sets (reqs [k, 32], meta [k, 32], payload), each grouped by gid, with no gid in two sets -> one set
    grouped by gid, its values packed 16-byte aligned in that order (the requests decoders' layout)"""
    reqs = np.concatenate([wire.to_records(p[0], abi.request_dtype) for p in parts])
    meta = np.concatenate([wire.to_records(p[1], abi.req_meta_dtype) for p in parts])
    vals = [bytes(p[2][int(r["payload_off"]): int(r["payload_off"]) + int(r["payload_len"])])
            for p in ((a, b, c.cpu().numpy()) for a, b, c in parts) for r in wire.to_records(p[0], abi.request_dtype)]
    order = np.argsort(reqs["gid"], kind="stable")
    reqs, meta, vals = reqs[order], meta[order], [vals[i] for i in order]
    arena, off = bytearray(), []
    for v in vals:
        off.append(len(arena))
        arena += v + bytes(-len(v) % 16)
    reqs["payload_off"] = off
    return dev_recs(reqs, 32), dev_recs(meta, 32), torch.from_numpy(np.frombuffer(bytes(arena) + bytes(16), np.uint8)
                                                                    .copy()).to(DEV), len(arena)


@pytest.mark.parametrize("G", [512, 100_000])
def test_three_nodes_sweeping_replies_and_forwards_equal_one_oracle_engine(cuda_lib, oracle_lib, G):
    MEMBERS = (100, 101, 102)
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    descs = np.zeros(G, abi.group_desc_dtype)
    descs["gid"] = np.arange(G)
    descs["name_hash"] = [abi.java_string_hash(s) for s in names]
    descs["n_members"] = 3
    descs["members"][:, :3] = MEMBERS
    descs["init_mode"] = abi.INIT_BATCH
    coord = np.array([coordinator_of(s, list(MEMBERS)) for s in names])
    gids = np.nonzero(coord == 100)[0]
    common = dict(max_groups=G, window=8, max_group_size=3, max_batch_recs=4 * G, max_batch_payload=64 * G)
    A = Engine(cuda_lib, make_config(cuda_lib, n_lanes=1, lane_node=[100], **common))
    B = Engine(cuda_lib, make_config(cuda_lib, n_lanes=2, lane_node=[101, 102], **common))
    O = Engine(oracle_lib, make_config(oracle_lib, n_lanes=3, lane_node=[100, 101, 102], **common))
    for e in (A, B, O):
        e.create_groups(descs)
    for e in (A, B):
        wire.set_group_names(e, gids, [names[g] for g in gids])
    dA, dB = DevNode(A), DevNode(B)
    got = {100: [], 101: [], 102: []}
    want = {100: [], 101: [], 102: []}
    caps = {}
    rounds = 5
    rng = np.random.default_rng(G)
    client = []
    for r in range(rounds):
        per = rng.integers(1, 4, size=len(gids)) if r in (1, 3) else np.ones(len(gids), int)
        rg = np.repeat(gids, per)
        stop = np.zeros(len(rg), bool) if r < rounds - 1 else (rg % 7 == 0)
        client.append(make_requests(rg, payload_len=5 + r, seed=3, round_no=r, entry_lane=1, entry_node=101,
                                    stop_mask=stop))

    def b_forwards(r):
        """B (node 101): round r's client bytes -> proposals -> FORWARD, on the device"""
        reqs, pay = client[r]
        pk = [wire.encode_request(wire.Request(names[int(q["gid"])], 0, int(q["req_id"]),
                                               bytes(pay[int(q["payload_off"]): int(q["payload_off"]) + int(q["payload_len"])]),
                                               stop=bool(int(q["flags"]) & abi.F_STOP), client=("10.1.2.3", 4567)))
              for q in reqs]
        arena, refs = request_arena([(b, 101) for b in pk])
        d = wire.decode_requests_device(B, arena, refs, NOW_MS, caps.get("breq", (1, 16)))
        caps["breq"] = d.sizes
        st = torch.empty(d.sizes[0], dtype=torch.int32, device=DEV)
        wire.propose_device_heads(B, d.reqs, d.sizes[0], d.payload, d.sizes[1], st,
                                  torch.empty((d.sizes[0], 48), dtype=torch.uint8, device=DEV),
                                  torch.empty(d.sizes[0], dtype=torch.int32, device=DEV), dB.ctl())
        assert (st == abi.RS_FORWARD).all()
        return d.reqs, d.meta, d.sizes[0], st, d.payload, []

    def a_takes(rep_b, fwd):
        """B's sweep -> A: (replies, their count, requests (reqs, meta, payload, payload bytes) or None)"""
        s = wire.encode_json_sweep_device(B, rep_b, 0 if rep_b is None else rep_b.shape[0], None, None, 0,
                                          *(fwd if fwd is not None else (None, None, 0, None, None, [])),
                                          caps.get("sweep", (1 << 16, 4)))
        caps["sweep"] = s.sizes
        if fwd is not None:
            assert (s.rstatus_reqs == abi.WE_SENT).all()
        assert (ref_nodes(s.refs) == 100).all()
        j = wire.decode_json_device(A, s.out, s.refs, caps.get("json", (1, 1, 1)))
        caps["json"] = j.sizes
        wrapped = j.status == abi.WS_OK
        assert ((j.status == abi.WS_OK) | (j.status == abi.WS_UNHANDLED)).all()
        if fwd is None:
            return j.replies, j.sizes[1], None
        jr = wire.decode_json_requests_device(A, s.out, s.refs, j.members, j.sizes[0], NOW_MS, (1, 16))
        lone = s.refs[~wrapped].contiguous()
        parts = [(jr.reqs, jr.meta, jr.payload)]
        if lone.shape[0]:
            lr = wire.decode_requests_device(A, s.out, lone, NOW_MS, (1, 16))
            assert (lr.status == abi.WS_OK).all()
            parts.append((lr.reqs, lr.meta, lr.payload))
        return j.replies, j.sizes[1], repack(parts)

    _, _, nxt = a_takes(None, b_forwards(0))
    for r in range(rounds):
        reqs, pay = client[r]
        a_reqs, a_meta, a_pay, a_pay_bytes = nxt
        n = a_reqs.shape[0]
        assert n == len(reqs)
        st = torch.empty(n, dtype=torch.int32, device=DEV)
        acc = torch.empty((n, 48), dtype=torch.uint8, device=DEV)
        heads = torch.empty(n, dtype=torch.int32, device=DEV)
        ctl_p = dA.ctl()
        wire.propose_device_heads(A, a_reqs, n, a_pay, a_pay_bytes, st, acc, heads, ctl_p)
        ea = wire.encode_accepts_device(A, acc, ctl_p.data_ptr(), n, heads, a_reqs, a_meta, n, a_pay,
                                        caps.get("acc", (64, 1)))
        caps["acc"] = ea.sizes
        na = int(ctl_p[0].item())
        acc_o, blob_o, st_o = O.propose(reqs, pay)
        assert np.array_equal(st.cpu().numpy(), st_o) and na == len(acc_o)
        sel = ref_nodes(ea.refs) == 101
        db = wire.decode_batch_device(B, ea.out.clone(), ea.refs[sel].contiguous(), caps.get("dacc", (1, 16, 1, 1)))
        caps["dacc"] = db.sizes
        assert db.sizes[0] == na and (db.status == abi.WS_OK).all()
        ctl_b, extra_b = dB.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_b = dB.accepts(db, ctl_b, extra_b)
        # B's sweep: this round's replies and the next round's forwards
        rep_j, n_rep_j, nxt = a_takes(rep_b, b_forwards(r + 1) if r + 1 < rounds else None)
        da2 = wire.decode_batch_device(A, ea.out.clone(), ea.refs[sel].contiguous(), caps.get("aacc", (1, 16, 1, 1)))
        caps["aacc"] = da2.sizes
        ctl_a1, extra_a1 = dA.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_a = dA.accepts(da2, ctl_a1, extra_a1)
        rep_o, _ = O.handle_accepts(acc_o, blob_o)
        ctl_a = dA.ctl()
        dec_a = torch.empty((4 * len(reqs), 32), dtype=torch.uint8, device=DEV)
        dA.replies(rep_a[:na], na, dec_a, ctl_a)
        dA.replies(rep_j, n_rep_j, dec_a, ctl_a)
        dec_o = O.handle_accept_replies(rep_o)
        enc2 = wire.encode_decisions_device(A, dec_a, ctl_a.data_ptr() + 4, dec_a.shape[0], caps.get("dec", (64, 1)))
        caps["dec"] = enc2.sizes
        n_dec = int(ctl_a[1].item())
        assert n_dec == len(dec_o)
        sel = ref_nodes(enc2.refs) == 101
        d3 = wire.decode_batch_device(B, enc2.out.clone(), enc2.refs[sel].contiguous(), caps.get("com", (1, 16, 1, 1)))
        caps["com"] = d3.sizes
        ctl_ax, extra_a = dA.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        ex_a = dA.decisions(dec_a, n_dec, extra_a, ctl_ax)
        ctl_bx = dB.ctl()
        extra_b.zero_()
        ex_b = dB.decisions(d3.decisions, d3.sizes[3], extra_b, ctl_bx)
        ex_o, x_o = O.handle_decisions(dec_o)
        for dct, ex in ((got, by_node(exec_and_extra(ex_a, extra_a, ctl_ax), [100])),
                        (got, by_node(exec_and_extra(ex_b, extra_b, ctl_bx), [101, 102])),
                        (want, by_node(np.concatenate([ex_o, x_o]), [100, 101, 102]))):
            for node, v in ex.items():
                dct[node].extend(v)
    for node in (100, 101, 102):
        assert got[node] == want[node] and len(want[node]) > 0
    for eng, lane, olane in ((A, 0, 0), (B, 0, 1), (B, 1, 2)):
        ra, ro = eng.dump_rows(gids, lane), O.dump_rows(gids, olane)
        for f in abi.row_dtype.names:
            if f != "lane":
                assert np.array_equal(ra[f], ro[f]), f
    for e in (A, B, O):
        e.close()
