"""GPU: the coordinator's side of the phase-2 wire on the device (gpx_wire_decode_requests_device,
gpx_propose_device_heads, gpx_wire_encode_accepts_device).

* Heads: gpx_propose_device_heads writes what gpx_propose_device writes, and every head names the request that starts
  its ACCEPT's slot: same gid, GPX_MK_HEAD-style status = the slot, nreq consecutive requests.
* Host codec: the two wire calls give the bytes the host codec and its restatement say, on torch's default stream and a
  side stream; GPX_ERANGE leaves 0xAB-filled outputs untouched.
* Two hosts, nothing on the host: node 100 (engine A) turns client REQUEST packets into ACCEPT packets on the device;
  nodes 101 and 102 (engine B) accept and reply on the device; A tallies and sends decisions.  EXEC records, rows and
  counters equal one oracle engine hosting all three nodes.
* PCIe: a coordinator chain copies a few bytes of counts between host and device, however large the batch.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import Engine, abi, group_descs_fast, make_config, make_requests
from test_wire_dev_gpu import by_node, world_engine
from test_wire_device_gpu import DevNode, dev_recs, dptr, exec_and_extra, host_bytes, pcie_bytes, ref_nodes
from wire_coord_cases import (NOW_MS, check_requests, expected_accepts, malformed_request_packets, random_accepts,
                              random_request_packets)
from wire_dev_cases import random_world

from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu

DEV = "cuda"


def request_arena(pkts):
    """[(bytes, node, ...)] -> device (arena, refs) with each packet's receiving node"""
    arena, refs = wire.pack_packets([p[0] for p in pkts])
    refs["node"] = [p[1] for p in pkts]
    return (torch.from_numpy(arena.copy() if len(arena) else np.zeros(1, np.uint8)).to(DEV),
            torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16).copy()).to(DEV))


def same_accepts(a, b):
    """the same ACCEPTs up to what k_propose leaves to the order its threads run in: the order of blocks' reservations
    and the blob offset of a batched slot (an atomicAdd on ctl->blob1_used)"""
    def key(x):
        x = x.copy()
        x["payload_off"][x["nreq"] > 1] = 0
        return np.sort(x.view(np.dtype((np.void, 48))))
    return np.array_equal(key(a), key(b))


def heads_case(cuda_lib, world, reqs, pay):
    """gpx_propose_device and gpx_propose_device_heads on two engines in the same state"""
    outs = []
    for with_heads in (False, True):
        e = world_engine(cuda_lib, world, window=2)
        d_reqs, d_pay = dev_recs(reqs, 32), torch.from_numpy(pay.copy()).to(DEV)
        got = []
        for rnd in range(3):  # the window fills: backpressure in the later rounds
            n = len(reqs)
            st = torch.full((n,), 0x55, dtype=torch.int32, device=DEV)
            acc = torch.full((n, 48), 0xAB, dtype=torch.uint8, device=DEV)
            ctl = torch.zeros(8, dtype=torch.int32, device=DEV)
            heads = torch.full((n,), 0x7AB, dtype=torch.int32, device=DEV)
            if with_heads:
                wire.propose_device_heads(e, d_reqs, n, d_pay, len(pay), st, acc, heads, ctl)
            else:
                e.L.check(e.L.fn("propose_device")(e.handle, dptr(d_reqs), dptr(d_pay), C.c_uint64(len(pay)),
                                                   C.c_uint32(n), dptr(st), dptr(acc), dptr(ctl), wire.stream_handle()))
            torch.cuda.synchronize()
            got.append((host_bytes(st), host_bytes(acc), host_bytes(ctl), heads.cpu().numpy().view(np.uint32)))
        rows = [e.dump_rows(list(world.groups), l).tobytes() for l in range(len(world.lanes))]
        outs.append((got, rows, e.counters()))
        e.close()
    (plain, rows0, c0), (withh, rows1, c1) = outs
    assert rows0 == rows1 and c0 == c1
    n_heads = 0
    for (st0, acc0, ctl0, _), (st1, acc1, ctl1, heads) in zip(plain, withh):
        assert st0 == st1 and ctl0 == ctl1
        na = int(np.frombuffer(ctl1, np.uint32)[0])
        acc = np.frombuffer(acc1, abi.accept_dtype)[:na]
        assert same_accepts(np.frombuffer(acc0, abi.accept_dtype)[:na], acc)
        assert acc1[48 * na:] == acc0[48 * na:]
        status = np.frombuffer(st1, np.int32)
        for k, a in enumerate(acc):
            h = int(heads[k])
            if int(a["flags"]) & abi.F_VOID:
                assert h == 0xFFFFFFFF
                continue
            nreq = int(a["nreq"])
            assert h + nreq <= len(reqs) and (reqs["gid"][h: h + nreq] == a["gid"]).all()
            assert status[h] == a["slot"] and int(reqs[h]["req_id"]) == int(a["req_id"])
            assert (status[h + 1: h + nreq] == -1).all()  # GPX_RS_BATCHED
            n_heads += 1
        assert (heads[na:] == 0x7AB).all()
    return n_heads, [np.frombuffer(g[0], np.int32) for g in withh]


def test_heads_match_propose_device_and_name_each_slot(cuda_lib):
    rng = np.random.default_rng(3)
    world = random_world(rng, 80)
    gids = sorted(int(g) for g in world.groups for _ in range(int(rng.integers(1, 5))))
    lanes = [world.lane_of(world.groups[g][2][0]) for g in gids]
    reqs, pay = make_requests(np.array(gids), payload_len=7, seed=5)
    reqs["flags"] = [((0 if l is None else l) << 8) for l in lanes]
    stop = rng.integers(0, 6, size=len(reqs)) == 0  # a STOP refuses what follows it (PCS.propose :235-239)
    reqs["flags"] |= np.where(stop, abi.F_STOP, 0).astype(np.uint32)
    n_heads, statuses = heads_case(cuda_lib, world, reqs, pay)
    assert n_heads > 0
    seen = set(int(x) for s in statuses for x in s)
    assert -4 in seen and -3 in seen  # backpressure, refused after a STOP


def coord_bytes_case(cuda_lib, seed, stream=None):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 60)
    e = world_engine(cuda_lib, world)
    pkts = random_request_packets(rng, world, 600)
    arena, refs = request_arena(pkts)
    d = wire.decode_requests_device(e, arena, refs, NOW_MS, (4, 64), stream)
    torch.cuda.synchronize()
    check_requests(world, pkts, (d.status.cpu().numpy(), wire.to_records(d.reqs, abi.request_dtype),
                                 wire.to_records(d.meta, abi.req_meta_dtype), d.payload.cpu().numpy()))
    cases = malformed_request_packets(world)
    arena, refs = request_arena(cases)
    d = wire.decode_requests_device(e, arena, refs, NOW_MS, (1, 16), stream)
    torch.cuda.synchronize()
    assert d.status.cpu().tolist() == [c[2] for c in cases]
    acc, heads, reqs, meta, pay = random_accepts(rng, world, 40)
    bad = np.nonzero((acc["flags"] & abi.F_VOID) == 0)[0][0]
    heads[bad] = len(reqs) + 3
    cnt = torch.tensor([len(acc) - 2], dtype=torch.int32, device=DEV)
    pad = np.concatenate([acc, acc[:5]])
    hp = np.concatenate([heads, heads[:5]])
    got = wire.encode_accepts_device(e, dev_recs(pad, 48), cnt.data_ptr(), len(pad),
                                     torch.from_numpy(hp.view(np.int32).copy()).to(DEV), dev_recs(reqs, 32),
                                     dev_recs(meta, 32), len(reqs), torch.from_numpy(pay.copy()).to(DEV), (64, 1),
                                     stream)
    torch.cuda.synchronize()
    est, exp = expected_accepts(world, set(world.groups), acc, heads, reqs, meta, pay, count=len(acc) - 2)
    assert host_bytes(got.rstatus[: len(acc) - 2]) == est.tobytes()
    assert wire.unpack_packets(got.out.cpu().numpy(), wire.to_records(got.refs, abi.wire_ref_dtype)) == exp
    assert abi.WE_BAD_HEAD in est.tolist() and abi.WE_SENT in est.tolist()
    e.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_wire_calls_give_the_host_codec_bytes(cuda_lib, seed):
    coord_bytes_case(cuda_lib, seed)


def test_wire_calls_on_a_side_stream(cuda_lib):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        coord_bytes_case(cuda_lib, 3, side)
    torch.cuda.current_stream().wait_stream(side)


def test_too_small_outputs_are_erange_and_stay_untouched(cuda_lib):
    rng = np.random.default_rng(4)
    world = random_world(rng, 40)
    e = world_engine(cuda_lib, world)
    pkts = random_request_packets(rng, world, 300)
    arena, refs = request_arena(pkts)
    full = wire.decode_requests_device(e, arena, refs, NOW_MS, (1, 16))
    need = list(full.sizes)
    st = wire.stream_handle()
    for caps in ([need[0] - 1, need[1]], [need[0], need[1] - 1]):
        outs = [torch.full((caps[0] * 32,), 0xAB, dtype=torch.uint8, device=DEV) for _ in range(2)]
        pay = torch.full((caps[1],), 0xAB, dtype=torch.uint8, device=DEV)
        nq, nb = C.c_uint32(caps[0]), C.c_uint64(caps[1])
        sts = torch.empty(len(pkts), dtype=torch.int32, device=DEV)
        rc = e.L.fn("wire_decode_requests_device")(e.handle, C.c_uint32(len(pkts)), dptr(arena),
                                                   C.c_uint64(arena.numel()), dptr(refs), C.c_int64(NOW_MS),
                                                   dptr(sts), dptr(outs[0]), dptr(outs[1]), C.byref(nq), dptr(pay),
                                                   C.byref(nb), st)
        torch.cuda.synchronize()
        assert rc == abi.GPX_ERANGE and [nq.value, nb.value] == need
        assert all((o == 0xAB).all() for o in outs) and (pay == 0xAB).all()
    acc, heads, reqs, meta, pay = random_accepts(rng, world, 30)
    args = (dev_recs(acc, 48), None, len(acc), torch.from_numpy(heads.view(np.int32).copy()).to(DEV),
            dev_recs(reqs, 32), dev_recs(meta, 32), len(reqs), torch.from_numpy(pay.copy()).to(DEV))
    full = wire.encode_accepts_device(e, *args, (1, 1))
    torch.cuda.synchronize()
    need = list(full.sizes)
    for caps in ([need[0] - 1, need[1]], [need[0], need[1] - 1]):
        out = torch.full((caps[0],), 0xAB, dtype=torch.uint8, device=DEV)
        rf = torch.full((caps[1] * 16,), 0xAB, dtype=torch.uint8, device=DEV)
        rst = torch.full((len(acc),), 0xAB, dtype=torch.uint8, device=DEV)
        nb, nr = C.c_uint64(caps[0]), C.c_uint32(caps[1])
        rc = e.L.fn("wire_encode_accepts_device")(e.handle, dptr(args[0]), None, C.c_uint32(len(acc)), dptr(args[3]),
                                                  dptr(args[4]), dptr(args[5]), C.c_uint32(len(reqs)), dptr(args[7]),
                                                  dptr(rst), dptr(out), C.byref(nb), dptr(rf), C.byref(nr), st)
        torch.cuda.synchronize()
        assert rc == abi.GPX_ERANGE and [nb.value, nr.value] == need
        assert (out == 0xAB).all() and (rf == 0xAB).all() and host_bytes(rst) == host_bytes(full.rstatus)
    e.close()


# ---- two hosts, nothing on the host ----------------------------------------------------------------------------------
@pytest.mark.parametrize("R,window", [(3, 8), (5, 1), (3, 1), (5, 8)])
def test_two_hosts_from_request_bytes_equal_one_oracle_engine(cuda_lib, oracle_lib, R, window):
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
    gids = np.nonzero(coord == 100)[0]
    common = dict(max_groups=G, window=window, max_group_size=R, max_batch_recs=4 * G)
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
    rng = np.random.default_rng(R * 10 + window)
    for r in range(rounds):
        # several requests per group in some rounds (batched slots), STOPs in the last round
        per = rng.integers(1, 4, size=len(gids)) if r in (1, 3) and window > 1 else np.ones(len(gids), int)
        rg = np.repeat(gids, per)
        stop = np.zeros(len(rg), bool) if r < rounds - 1 else (rg % 7 == 0)
        reqs, pay = make_requests(rg, payload_len=5 + r, seed=3, round_no=r, entry_lane=0, entry_node=100,
                                  stop_mask=stop)
        client = [wire.encode_request(wire.Request(names[int(q["gid"])], 0, int(q["req_id"]),
                                                   bytes(pay[int(q["payload_off"]): int(q["payload_off"]) + int(q["payload_len"])]),
                                                   stop=bool(int(q["flags"]) & abi.F_STOP), client=("10.1.2.3", 4567)))
                  for q in reqs]
        arena, refs = request_arena([(b, 100) for b in client])
        # A: client bytes -> proposals -> ACCEPT bytes, on the device
        d = wire.decode_requests_device(A, arena, refs, NOW_MS, caps.get("req", (1, 16)))
        caps["req"] = d.sizes
        assert d.sizes[0] == len(reqs)
        n = d.sizes[0]
        st = torch.empty(n, dtype=torch.int32, device=DEV)
        acc = torch.empty((n, 48), dtype=torch.uint8, device=DEV)
        heads = torch.empty(n, dtype=torch.int32, device=DEV)
        ctl_p = dA.ctl()
        wire.propose_device_heads(A, d.reqs, n, d.payload, d.sizes[1], st, acc, heads, ctl_p)
        ea = wire.encode_accepts_device(A, acc, ctl_p.data_ptr(), n, heads, d.reqs, d.meta, n, d.payload,
                                        caps.get("acc", (64, 1)))
        caps["acc"] = ea.sizes
        na = int(ctl_p[0].item())
        acc_o, blob_o, st_o = O.propose(reqs, pay)
        assert np.array_equal(st.cpu().numpy(), st_o) and na == len(acc_o)
        assert (ea.rstatus[:na] == abi.WE_SENT).all() and ea.sizes[1] == na * (R - 1)
        # B: ACCEPT bytes addressed to node 101 (B serves 101 and 102: one copy)
        sel = ref_nodes(ea.refs) == 101
        db = wire.decode_batch_device(B, ea.out.clone(), ea.refs[sel].contiguous(), caps.get("dacc", (1, 16, 1, 1)))
        caps["dacc"] = db.sizes
        assert db.sizes[0] == na and (db.status == abi.WS_OK).all()
        ctl_b, extra_b = dB.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_b = dB.accepts(db, ctl_b, extra_b)
        enc = wire.encode_replies_device(B, rep_b, rep_b.shape[0], caps.get("rep", (64, 1)))
        caps["rep"] = enc.sizes
        # A: its own copy of the ACCEPT bytes (the encoder indexes none for a local lane: decode the stored packets)
        da = wire.decode_batch_device(A, ea.out.clone(), ea.refs[sel].contiguous(), caps.get("aacc", (1, 16, 1, 1)))
        caps["aacc"] = da.sizes
        assert da.sizes[0] == na and (da.status == abi.WS_OK).all()
        ctl_a1, extra_a1 = dA.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_a = dA.accepts(da, ctl_a1, extra_a1)
        rep_o, _ = O.handle_accepts(acc_o, blob_o)
        ctl_a = dA.ctl()
        dec_a = torch.empty((4 * len(rg), 32), dtype=torch.uint8, device=DEV)
        dA.replies(rep_a[:na], na, dec_a, ctl_a)
        d2 = wire.decode_batch_device(A, enc.out.clone(), enc.refs.clone(), caps.get("ab", (1, 16, 1, 1)))
        caps["ab"] = d2.sizes
        assert (d2.status == abi.WS_OK).all()
        dA.replies(d2.replies, d2.sizes[2], dec_a, ctl_a)
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
    ca, cb, co = A.counters(), B.counters(), O.counters()
    for k in ("decisions_made", "executed", "stops_executed", "accepts_handled", "replies_handled"):
        assert ca[k] + cb[k] == co[k], k
    for e in (A, B, O):
        e.close()


# ---- PCIe traffic of a coordinator chain ----------------------------------------------------------------------------
def test_a_coordinator_chain_moves_no_records_over_pcie(cuda_lib):
    got = {}
    for G in (10_000, 100_000):
        e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=1, lane_node=[100], window=8,
                                         max_batch_recs=G, max_batch_payload=16 * G, log_ring_bytes=1 << 20))
        e.create_groups(group_descs_fast(G, members=(100, 101, 102)))
        wire.set_group_names(e, np.arange(G, dtype=np.uint32), [f"NoopPaxosApp{i}" for i in range(G)])
        node = DevNode(e)
        st = torch.empty(G, dtype=torch.int32, device=DEV)
        acc = torch.empty((G, 48), dtype=torch.uint8, device=DEV)
        heads = torch.empty(G, dtype=torch.int32, device=DEV)

        def chain(arena, refs):
            d = wire.decode_requests_device(e, arena, refs, NOW_MS, (G, 16 * G))
            ctl = node.ctl()
            wire.propose_device_heads(e, d.reqs, d.sizes[0], d.payload, d.sizes[1], st, acc, heads, ctl)
            return wire.encode_accepts_device(e, acc, ctl.data_ptr(), d.sizes[0], heads, d.reqs, d.meta, d.sizes[0],
                                              d.payload, (256 * G, 2 * G))

        def packets(r):
            return request_arena([(wire.encode_request(wire.Request(f"NoopPaxosApp{i}", 0, r * G + i, b"12345678")), 100)
                                  for i in range(G)])

        out = chain(*packets(0))  # warm-up: the scratch grows here
        torch.cuda.synchronize()
        assert out.sizes[1] > 0
        arena, refs = packets(1)  # the caller's upload, outside the chain
        b, seen, out = pcie_bytes(lambda: chain(arena, refs))
        assert out.sizes[1] > 0 and seen > 0
        got[G] = b
        e.close()
    assert got[10_000] <= 4096 and got[100_000] <= got[10_000], got
