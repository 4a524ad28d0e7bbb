"""GPU: forwarding between nodes on the device (gpx_wire_encode_forwards_device, gpx_wire_decode_json_requests_device).

* Parity at 100 K groups, on torch's default stream and on a side stream: the forwards a non-coordinator's propose
  leaves are the packets the restatement of PISM.handleProposal feeds gpx_wire_encode_request, and the emulated kernel's
  (tests/emu/wire_fwd_emu.cpp); a Java peer's forwards as JSON members of wrappers decode to what the byte decoder and
  the emulated kernels make of them.  GPX_ERANGE leaves 0xAB-filled outputs untouched.
* Three nodes, nothing on the host: client REQUEST packets arrive at node 101 (engine B, lanes 101 and 102) for groups
  node 100 (engine A) coordinates; B's forwards go from bytes to bytes on the device, A decodes them, proposes, encodes
  ACCEPTs and the round completes over the device wire calls.  EXEC records and rows equal one oracle engine hosting
  all three nodes with the requests entered at node 101's lane.  The same forwards as JSON members of
  BATCHED_PAXOS_PACKETs (packets_json) give A the same proposals.
* PCIe: the forward chain copies a few bytes of counts between host and device, however large the batch."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import Engine, abi, group_descs_fast, make_config, make_requests
from test_wire_coord_gpu import request_arena
from test_wire_dev import Emu
from test_wire_dev_gpu import by_node
from test_wire_device_gpu import DevNode, dev_recs, dptr, exec_and_extra, host_bytes, pcie_bytes, ref_nodes
from test_wire_forward import decode_json_requests as emu_decode_json_requests
from test_wire_forward import decode_members as emu_decode_members
from test_wire_forward import emu  # noqa: F401  (the emulated kernels, a module fixture)
from test_wire_forward import encode_forwards as emu_encode_forwards
from wire_coord_cases import NOW_MS
from wire_dev_cases import World
from wire_fwd_cases import Rows, as_request, expected_forwards, request_member, wrapper

from gigapaxos_b200 import packets_json as pj
from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu

DEV = "cuda"
MEMBERS = (100, 101, 102)


def engine_rows(e: Engine, gids, G, cfg) -> Rows:
    """the rows k_wire_fwd reads, from gpx_dump_rows, and the engine's batching settings"""
    rows = Rows(e.n_lanes, G, batching=cfg.batching_enabled, max_batch_size=cfg.max_batch_size,
                size_est=cfg.request_size_estimate, max_batch_bytes=cfg.max_batch_bytes)
    rows.aux[:] = abi.ST_STOPPED
    for l in range(e.n_lanes):
        r = e.dump_rows(gids, l)
        g = r["gid"].astype(np.int64)
        rows.acc[l, g, 1], rows.acc[l, g, 2] = r["acc_bnum"], r["acc_bcoord"]
        rows.aux[l, g] = r["state"]
        rows.coord[l, g, 0], rows.coord[l, g, 1] = r["coord_bnum"], r["coord_bcoord"]
        rows.coord[l, g, 3] = (r["coord_exists"] != 0) | ((r["coord_active"] != 0) << 1)
    return rows


def alike_emu(lib, world: World, unnamed) -> Emu:
    """an emulated engine of the world's groups, which all have the members MEMBERS (one interned member set), named
    but for `unnamed`"""
    x = Emu.__new__(Emu)
    x.lib, x.world = lib, world
    G = max(world.groups) + 1
    lanes = np.array(world.lanes, np.int32)
    x.h = C.c_void_p(lib.emu_wire_new(G, len(lanes), lanes.ctypes.data_as(C.c_void_p)))
    gids, m = np.arange(G, dtype=np.uint32), np.array(MEMBERS, np.int32)
    assert lib.emu_wire_groups_alike(x.h, C.c_uint32(G), gids.ctypes.data_as(C.c_void_p), C.c_uint32(len(m)),
                                     m.ctypes.data_as(C.c_void_p)) == 0
    x.set_names([g for g in range(G) if g not in unnamed])
    return x


def forward_world(G, lane_node=(101,)):
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    cfg_kw = dict(max_groups=G, n_lanes=len(lane_node), lane_node=list(lane_node), window=8, max_batch_recs=4 * G,
                  max_batch_payload=64 * G, log_ring_bytes=1 << 24, max_batch_size=3)
    return names, World({g: (names[g], 0, list(MEMBERS)) for g in range(G)}, lanes=lane_node), cfg_kw


def client_requests(rng, G, names, entry_lane=0):
    """1-4 requests per group, with meta: addresses, flags, forward counts (3 ping-pongs once forwarded)"""
    per = rng.integers(1, 5, size=G)
    gids = np.repeat(np.arange(G), per)
    reqs, pay = make_requests(gids, payload_len=rng.integers(0, 24, size=len(gids)), seed=int(rng.integers(1 << 20)),
                              entry_lane=entry_lane, entry_node=101)
    meta = np.zeros(len(reqs), abi.req_meta_dtype)
    meta["client_ip"] = [10, 1, 2, 3]
    meta["client_port"] = rng.choice([0, 4567], size=len(reqs))
    meta["client_ip"][meta["client_port"] == 0] = 0
    meta["forward_count"] = rng.choice([0, 0, 0, 1, 3], size=len(reqs))
    meta["entry_time"] = rng.integers(0, 1 << 41, size=len(reqs))
    meta["flags"] = rng.choice([0, abi.RM_RETURN_VALUE], size=len(reqs))
    return reqs, meta, pay


def forwards_case(cuda_lib, emu_lib, seed, stream=None):
    rng = np.random.default_rng(seed)
    G = 100_000
    names, world, cfg_kw = forward_world(G)
    cfg = make_config(cuda_lib, **cfg_kw)
    e = Engine(cuda_lib, cfg)
    e.create_groups(group_descs_fast(G, members=MEMBERS))
    named = set(range(G)) - set(range(0, G, 97))
    wire.set_group_names(e, np.array(sorted(named), np.uint32), [names[g] for g in sorted(named)])
    reqs, meta, pay = client_requests(rng, G, names)
    n = len(reqs)
    d_reqs, d_meta, d_pay = dev_recs(reqs, 32), dev_recs(meta, 32), torch.from_numpy(pay.copy()).to(DEV)
    st = torch.empty(n, dtype=torch.int32, device=DEV)
    acc = torch.empty((n, 48), dtype=torch.uint8, device=DEV)
    heads = torch.empty(n, dtype=torch.int32, device=DEV)
    wire.propose_device_heads(e, d_reqs, n, d_pay, len(pay), st, acc, heads, torch.zeros(8, dtype=torch.int32,
                                                                                        device=DEV), stream)
    down = [102]
    out = wire.encode_forwards_device(e, d_reqs, d_meta, n, st, d_pay, down, (1, 1), stream)
    torch.cuda.synchronize()
    status = st.cpu().numpy()
    assert (status == abi.RS_FORWARD).sum() > n // 2
    rows = engine_rows(e, np.arange(G, dtype=np.uint32), G, cfg)
    got = wire.unpack_packets(out.out.cpu().numpy(), wire.to_records(out.refs, abi.wire_ref_dtype))
    rst = out.rstatus.cpu().numpy()
    est, exp = expected_forwards(world, named, rows, reqs, meta, status, pay, down)
    assert rst.tolist() == est.tolist() and got == exp
    assert {abi.WE_SENT, abi.WE_VOID, abi.WE_ELECT, abi.WE_NO_NAME} <= set(rst.tolist())
    assert {node for _, node, _ in got} == {100}  # 102 is down: the next member after it is 100
    # the emulated kernel on the same state
    x = alike_emu(emu_lib, world, set(range(0, G, 97)))
    rst_x, got_x = emu_encode_forwards(x, rows, reqs, meta, status, pay, down)
    assert rst_x.tolist() == rst.tolist() and got_x == got
    # the same requests as a Java peer's forwards, JSON members of wrappers received at node 101
    sel = [q for q in range(0, n, 7)]
    pk = [(wire.encode_request(as_request(world, reqs[q], meta[q], pay)), 101, as_request(world, reqs[q], meta[q], pay))
          for q in sel]
    members = [request_member(p[2], rng) for p in pk]
    wraps = [wrapper(members[i: i + 1000]) for i in range(0, len(members), 1000)]
    arena, refs = request_arena([(w, 101) for w in wraps])
    j = wire.decode_json_device(e, arena, refs, (1, 1, 1), stream)
    jr = wire.decode_json_requests_device(e, arena, refs, j.members, j.sizes[0], NOW_MS, (1, 16), stream)
    barena, brefs = request_arena([(p[0], 101) for p in pk])
    b = wire.decode_requests_device(e, barena, brefs, NOW_MS, (1, 16), stream)
    torch.cuda.synchronize()
    assert (j.status == abi.WS_OK).all() and j.sizes[0] == len(pk)
    assert host_bytes(jr.status) == host_bytes(b.status) and (jr.status == abi.WS_OK).sum() > len(pk) // 2
    assert host_bytes(jr.reqs) == host_bytes(b.reqs) and host_bytes(jr.meta) == host_bytes(b.meta)
    assert host_bytes(jr.payload) == host_bytes(b.payload)
    a_np, r_np = arena.cpu().numpy(), refs.cpu().numpy().reshape(-1).view(abi.wire_ref_dtype).copy()
    _, mem = emu_decode_members(x, a_np, r_np, len(a_np))
    rc, st_x, rq_x, mt_x, pay_x, _ = emu_decode_json_requests(x, a_np, r_np, len(a_np), mem)
    assert rc == 0 and st_x.tobytes() == host_bytes(jr.status)
    assert rq_x.tobytes() == host_bytes(jr.reqs) and mt_x.tobytes() == host_bytes(jr.meta)
    assert pay_x.tobytes() == host_bytes(jr.payload)
    x.close()
    return e, (d_reqs, d_meta, n, st, d_pay, down), (arena, refs, j)


def test_forwards_match_the_host_codec_and_the_emulated_kernels(cuda_lib, emu):
    e, _, _ = forwards_case(cuda_lib, emu, 1)
    e.close()


def test_forwards_on_a_side_stream(cuda_lib, emu):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        e, _, _ = forwards_case(cuda_lib, emu, 2, side)
    torch.cuda.current_stream().wait_stream(side)
    e.close()


def test_too_small_outputs_are_erange_and_stay_untouched(cuda_lib, emu):
    e, fargs, (arena, refs, j) = forwards_case(cuda_lib, emu, 3)
    d_reqs, d_meta, n, st, d_pay, down = fargs
    full = wire.encode_forwards_device(e, *fargs, (1, 1))
    torch.cuda.synchronize()
    need = list(full.sizes)
    dn = np.array(down, np.int32)
    for caps in ([need[0] - 1, need[1]], [need[0], need[1] - 1]):
        out = torch.full((caps[0],), 0xAB, dtype=torch.uint8, device=DEV)
        rf = torch.full((caps[1] * 16,), 0xAB, dtype=torch.uint8, device=DEV)
        rst = torch.full((n,), 0xAB, dtype=torch.uint8, device=DEV)
        nb, nr = C.c_uint64(caps[0]), C.c_uint32(caps[1])
        rc = e.L.fn("wire_encode_forwards_device")(e.handle, dptr(d_reqs), dptr(d_meta), C.c_uint32(n), dptr(st),
                                                   dptr(d_pay), C.c_uint32(1), dn.ctypes.data_as(C.c_void_p),
                                                   dptr(rst), dptr(out), C.byref(nb), dptr(rf), C.byref(nr),
                                                   wire.stream_handle())
        torch.cuda.synchronize()
        assert rc == abi.GPX_ERANGE and [nb.value, nr.value] == need
        assert (out == 0xAB).all() and (rf == 0xAB).all() and host_bytes(rst) == host_bytes(full.rstatus)
    full = wire.decode_json_requests_device(e, arena, refs, j.members, j.sizes[0], NOW_MS, (1, 16))
    torch.cuda.synchronize()
    need = list(full.sizes)
    for caps in ([need[0] - 1, need[1]], [need[0], need[1] - 1]):
        outs = [torch.full((caps[0] * 32,), 0xAB, dtype=torch.uint8, device=DEV) for _ in range(2)]
        pay = torch.full((caps[1],), 0xAB, dtype=torch.uint8, device=DEV)
        nq, nb = C.c_uint32(caps[0]), C.c_uint64(caps[1])
        sts = torch.empty(j.sizes[0], dtype=torch.int32, device=DEV)
        rc = e.L.fn("wire_decode_json_requests_device")(e.handle, C.c_uint32(j.sizes[0]), dptr(arena),
                                                        C.c_uint64(arena.numel()), dptr(refs),
                                                        C.c_uint32(refs.shape[0]), dptr(j.members),
                                                        C.c_int64(NOW_MS), dptr(sts), dptr(outs[0]), dptr(outs[1]),
                                                        C.byref(nq), dptr(pay), C.byref(nb), wire.stream_handle())
        torch.cuda.synchronize()
        assert rc == abi.GPX_ERANGE and [nq.value, nb.value] == need
        assert all((o == 0xAB).all() for o in outs) and (pay == 0xAB).all()
    e.close()


# ---- three nodes, nothing on the host ---------------------------------------------------------------------------------
@pytest.mark.parametrize("window", [8, 1])
def test_three_nodes_forwarding_on_the_device_equal_one_oracle_engine(cuda_lib, oracle_lib, window):
    G = 512
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    descs = np.zeros(G, abi.group_desc_dtype)
    descs["gid"] = np.arange(G)
    descs["name_hash"] = [abi.java_string_hash(s) for s in names]
    descs["n_members"] = 3
    descs["members"][:, :3] = MEMBERS
    descs["init_mode"] = abi.INIT_BATCH
    coord = np.array([coordinator_of(s, list(MEMBERS)) for s in names])
    gids = np.nonzero(coord == 100)[0]
    common = dict(max_groups=G, window=window, max_group_size=3, max_batch_recs=4 * G)
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
    rng = np.random.default_rng(window)
    for r in range(rounds):
        per = rng.integers(1, 4, size=len(gids)) if r in (1, 3) and window > 1 else np.ones(len(gids), int)
        rg = np.repeat(gids, per)
        stop = np.zeros(len(rg), bool) if r < rounds - 1 else (rg % 7 == 0)
        reqs, pay = make_requests(rg, payload_len=5 + r, seed=3, round_no=r, entry_lane=1, entry_node=101,
                                  stop_mask=stop)
        client = [wire.encode_request(wire.Request(names[int(q["gid"])], 0, int(q["req_id"]),
                                                   bytes(pay[int(q["payload_off"]): int(q["payload_off"]) + int(q["payload_len"])]),
                                                   stop=bool(int(q["flags"]) & abi.F_STOP), client=("10.1.2.3", 4567)))
                  for q in reqs]
        # B (node 101): client bytes -> proposals -> FORWARD -> REQUEST bytes to node 100, on the device
        arena, refs = request_arena([(b, 101) for b in client])
        d = wire.decode_requests_device(B, arena, refs, NOW_MS, caps.get("breq", (1, 16)))
        caps["breq"] = d.sizes
        nb_ = d.sizes[0]
        st_b = torch.empty(nb_, dtype=torch.int32, device=DEV)
        wire.propose_device_heads(B, d.reqs, nb_, d.payload, d.sizes[1], st_b,
                                  torch.empty((nb_, 48), dtype=torch.uint8, device=DEV),
                                  torch.empty(nb_, dtype=torch.int32, device=DEV), dB.ctl())
        fw = wire.encode_forwards_device(B, d.reqs, d.meta, nb_, st_b, d.payload, [], caps.get("fwd", (64, 1)))
        caps["fwd"] = fw.sizes
        assert (st_b == abi.RS_FORWARD).all() and (fw.rstatus == abi.WE_SENT).all()
        assert (ref_nodes(fw.refs) == 100).all()
        # A (node 100): the forwards -> proposals, and the same forwards as a Java peer's JSON members
        fa, fr = fw.out.clone(), fw.refs.clone()
        fr.view(torch.int32).reshape(-1, 4)[:, 3] = 100  # the receiving node
        da = wire.decode_requests_device(A, fa, fr, NOW_MS, caps.get("areq", (1, 16)))
        caps["areq"] = da.sizes
        assert (da.status == abi.WS_OK).all() and da.sizes[0] == len(reqs)
        pk = wire.unpack_packets(fw.out.cpu().numpy(), wire.to_records(fw.refs, abi.wire_ref_dtype))
        jm = [_request_json_of(p[2]) for p in pk]
        wraps = [pj.batched_paxos_packet_json(jm[i: i + 100]) for i in range(0, len(jm), 100)]
        ja, jrf = request_arena([(w, 100) for w in wraps])
        j = wire.decode_json_device(A, ja, jrf, (1, 1, 1))
        jr = wire.decode_json_requests_device(A, ja, jrf, j.members, j.sizes[0], NOW_MS, (1, 16))
        assert (jr.status == abi.WS_OK).all() and host_bytes(jr.reqs) == host_bytes(da.reqs)
        assert host_bytes(jr.meta) == host_bytes(da.meta) and host_bytes(jr.payload) == host_bytes(da.payload)
        n = da.sizes[0]
        st = torch.empty(n, dtype=torch.int32, device=DEV)
        acc = torch.empty((n, 48), dtype=torch.uint8, device=DEV)
        heads = torch.empty(n, dtype=torch.int32, device=DEV)
        ctl_p = dA.ctl()
        wire.propose_device_heads(A, da.reqs, n, da.payload, da.sizes[1], st, acc, heads, ctl_p)
        ea = wire.encode_accepts_device(A, acc, ctl_p.data_ptr(), n, heads, da.reqs, da.meta, n, da.payload,
                                        caps.get("acc", (64, 1)))
        caps["acc"] = ea.sizes
        na = int(ctl_p[0].item())
        acc_o, blob_o, st_o = O.propose(reqs, pay)
        assert np.array_equal(st.cpu().numpy(), st_o) and na == len(acc_o)
        # B: ACCEPT bytes addressed to node 101; the round completes as between two hosts
        sel = ref_nodes(ea.refs) == 101
        db = wire.decode_batch_device(B, ea.out.clone(), ea.refs[sel].contiguous(), caps.get("dacc", (1, 16, 1, 1)))
        caps["dacc"] = db.sizes
        assert db.sizes[0] == na and (db.status == abi.WS_OK).all()
        ctl_b, extra_b = dB.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_b = dB.accepts(db, ctl_b, extra_b)
        enc = wire.encode_replies_device(B, rep_b, rep_b.shape[0], caps.get("rep", (64, 1)))
        caps["rep"] = enc.sizes
        da2 = wire.decode_batch_device(A, ea.out.clone(), ea.refs[sel].contiguous(), caps.get("aacc", (1, 16, 1, 1)))
        caps["aacc"] = da2.sizes
        ctl_a1, extra_a1 = dA.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_a = dA.accepts(da2, ctl_a1, extra_a1)
        rep_o, _ = O.handle_accepts(acc_o, blob_o)
        ctl_a = dA.ctl()
        dec_a = torch.empty((4 * len(rg), 32), dtype=torch.uint8, device=DEV)
        dA.replies(rep_a[:na], na, dec_a, ctl_a)
        d2 = wire.decode_batch_device(A, enc.out.clone(), enc.refs.clone(), caps.get("ab", (1, 16, 1, 1)))
        caps["ab"] = d2.sizes
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
    for e in (A, B, O):
        e.close()


def _request_json_of(packet: bytes) -> bytes:
    """the JSON form (packets_json.request_json) of a REQUEST packet the host codec reads back"""
    return pj.request_json(_parse_request(packet))


def _parse_request(b: bytes, at: int = 0):
    import struct
    n = b[at + 12]
    name = b[at + 13: at + 13 + n].decode("iso-8859-1")
    ver = struct.unpack(">i", b[at + 8: at + 12])[0]
    p = at + 13 + n
    rid, stop = struct.unpack(">qB", b[p: p + 9])
    p += 9
    cip, cport, lip, lport = b[p: p + 4], struct.unpack(">H", b[p + 4: p + 6])[0], b[p + 6: p + 10], \
        struct.unpack(">H", b[p + 10: p + 12])[0]
    p += 12
    entry, et, rv, fc, bc = struct.unpack(">iqBiB", b[p: p + 18])
    p += 18
    dl = struct.unpack(">i", b[p: p + 4])[0]
    p += 4 + dl
    vl = struct.unpack(">i", b[p: p + 4])[0]
    val = b[p + 4: p + 4 + vl]
    p += 4 + vl
    rl = struct.unpack(">i", b[p: p + 4])[0]
    p += 4 + rl
    nbat = struct.unpack(">i", b[p: p + 4])[0]
    p += 4
    subs = []
    for _ in range(nbat):
        ln = struct.unpack(">i", b[p: p + 4])[0]
        subs.append(_parse_request(b[p + 4: p + 4 + ln]))
        p += 4 + ln
    addr = lambda ip, port: (".".join(str(x) for x in ip), port) if port else None
    return wire.Request(name, ver, rid, val, stop=bool(stop), entry_replica=entry, entry_time=et,
                        client=addr(cip, cport), listen=addr(lip, lport), should_return=bool(rv), forward_count=fc,
                        broadcasted=bool(bc), batched=tuple(subs))


# ---- PCIe traffic of the forward chain ----------------------------------------------------------------------------
def test_the_forward_chain_moves_no_records_over_pcie(cuda_lib):
    got = {}
    for G in (10_000, 100_000):
        e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=1, lane_node=[101], window=8,
                                         max_batch_recs=G, max_batch_payload=16 * G, log_ring_bytes=1 << 20))
        e.create_groups(group_descs_fast(G, members=MEMBERS))
        wire.set_group_names(e, np.arange(G, dtype=np.uint32), [f"NoopPaxosApp{i}" for i in range(G)])
        node = DevNode(e)
        st = torch.empty(G, dtype=torch.int32, device=DEV)
        acc = torch.empty((G, 48), dtype=torch.uint8, device=DEV)
        heads = torch.empty(G, dtype=torch.int32, device=DEV)

        def chain(arena, refs):
            d = wire.decode_requests_device(e, arena, refs, NOW_MS, (G, 16 * G))
            wire.propose_device_heads(e, d.reqs, d.sizes[0], d.payload, d.sizes[1], st, acc, heads, node.ctl())
            return wire.encode_forwards_device(e, d.reqs, d.meta, d.sizes[0], st, d.payload, [], (256 * G, G))

        def packets(r):
            return request_arena([(wire.encode_request(wire.Request(f"NoopPaxosApp{i}", 0, r * G + i, b"12345678")), 101)
                                  for i in range(G)])

        out = chain(*packets(0))  # warm-up: the scratch grows here
        torch.cuda.synchronize()
        assert out.sizes[1] > G // 2
        arena, refs = packets(1)  # the caller's upload, outside the chain
        b, seen, out = pcie_bytes(lambda: chain(arena, refs))
        assert out.sizes[1] > G // 2 and seen > 0
        got[G] = b
        e.close()
    assert got[10_000] <= 4096 and got[100_000] <= got[10_000], got
