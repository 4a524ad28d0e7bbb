"""GPU: the device-buffer forms of the phase-2 wire calls (gpx_wire_decode_batch_device, gpx_wire_encode_*_device).

* Bytes: the cases of tests/test_wire_dev_gpu.py through the device forms and the host forms on one engine give
  byte-identical statuses, records, blobs, packet arenas, refs and rstatus -- on torch's default stream and on a side
  stream.
* GPX_ERANGE: an output one short returns the sizes needed and leaves every output untouched.
* Two hosts, records never on the host: engine A (node 100) and engine B (nodes 101, 102) exchange only packet arenas;
  B decodes, handles and encodes on the device, A tallies its own replies and the decoded remote ones on the device and
  encodes its decisions from the tally's device count.  EXEC records, rows and counters equal one oracle engine.
* No records over PCIe: an acceptor chain (decode -> accepts -> encode replies) moves a few bytes of counts between
  host and device, however large the batch.
"""
import ctypes as C
import json
import os
import tempfile

import numpy as np
import pytest
import torch

from helpers import Engine, abi, group_descs_fast, make_config, make_requests
from test_wire_dev_gpu import accept_packets, by_node, world_engine
from wire_dev_cases import malformed_packets, random_decisions, random_packets, random_replies, random_world

from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu

DEV = "cuda"


def dptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def dev_recs(a: np.ndarray, width: int):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(len(a), width).copy()).to(DEV)


def host_bytes(t) -> bytes:
    return t.detach().cpu().numpy().tobytes()


def same_decode(e, pkts, stream=None):
    status, acc, blob, rep, dec = wire.decode_batch(e, pkts)
    arena, refs = wire.device_packets(pkts)
    d = wire.decode_batch_device(e, arena, refs, (len(pkts), 64, 1, 1), stream)
    torch.cuda.synchronize()
    assert host_bytes(d.status) == status.tobytes()
    assert host_bytes(d.accepts) == acc.tobytes() and host_bytes(d.blob) == blob.tobytes()
    assert host_bytes(d.replies) == rep.tobytes() and host_bytes(d.decisions) == dec.tobytes()
    return d


def same_encode(host, dev):
    torch.cuda.synchronize()
    rst, arena, refs = host
    assert host_bytes(dev.rstatus) == rst.tobytes()
    assert host_bytes(dev.out) == arena.tobytes() and host_bytes(dev.refs) == refs.tobytes()


def same_bytes_case(cuda_lib, seed, stream=None):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 60)
    e = world_engine(cuda_lib, world)
    pkts, _ = random_packets(rng, world, 2000)
    d = same_decode(e, pkts, stream)
    assert min(d.sizes) > 0
    same_decode(e, [p for p, _ in malformed_packets(world)], stream)
    L = len(world.lanes)
    rep = random_replies(rng, world, 500, L)
    same_encode(wire.encode_replies(e, rep), wire.encode_replies_device(e, dev_recs(rep, 32), len(rep), (64, 1), stream))
    dec = random_decisions(rng, world, 800)
    same_encode(wire.encode_decisions(e, dec),
                wire.encode_decisions_device(e, dev_recs(dec, 32), None, len(dec), (64, 1), stream))
    # a device count: the records behind it are valid-looking but not counted
    pad = np.concatenate([dec[:500], random_decisions(rng, world, 100)])
    cnt = torch.tensor([500], dtype=torch.int32, device=DEV)
    got = wire.encode_decisions_device(e, dev_recs(pad, 32), cnt.data_ptr(), len(pad), (64, 1), stream)
    host = wire.encode_decisions(e, dec[:500])
    torch.cuda.synchronize()
    assert host_bytes(got.rstatus[:500]) == host[0].tobytes()
    assert host_bytes(got.out) == host[1].tobytes() and host_bytes(got.refs) == host[2].tobytes()
    e.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_device_forms_give_the_bytes_of_the_host_forms(cuda_lib, seed):
    same_bytes_case(cuda_lib, seed)


@pytest.mark.parametrize("seed", [1, 2])
def test_device_forms_on_a_side_stream(cuda_lib, seed):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # the inputs are made on the side stream too
        same_bytes_case(cuda_lib, seed, side)
    torch.cuda.current_stream().wait_stream(side)


def test_too_small_outputs_are_erange_and_stay_untouched(cuda_lib):
    rng = np.random.default_rng(4)
    world = random_world(rng, 40)
    e = world_engine(cuda_lib, world)
    pkts, _ = random_packets(rng, world, 500)
    status, acc, blob, rep, dec = wire.decode_batch(e, pkts)
    need = [len(acc), len(blob), len(rep), len(dec)]
    assert min(need) > 0
    arena, refs = wire.device_packets(pkts)
    fn = cuda_lib.fn("wire_decode_batch_device")
    st = wire.stream_handle()

    def decode(caps):
        outs = [torch.full((c * w,), 0xAB, dtype=torch.uint8, device=DEV) for c, w in zip(caps, (48, 1, 32, 32))]
        sts = torch.full((len(pkts),), -7, dtype=torch.int32, device=DEV)
        sz = [C.c_uint32(caps[0]), C.c_uint64(caps[1]), C.c_uint32(caps[2]), C.c_uint32(caps[3])]
        rc = fn(e.handle, C.c_uint32(len(pkts)), dptr(arena), C.c_uint64(arena.numel()), dptr(refs), dptr(sts),
                dptr(outs[0]), C.byref(sz[0]), dptr(outs[1]), C.byref(sz[1]), dptr(outs[2]), C.byref(sz[2]),
                dptr(outs[3]), C.byref(sz[3]), st)
        torch.cuda.synchronize()
        return rc, [s.value for s in sz], outs, sts

    shorts = [[c - (j == k) for j, c in enumerate(need)] for k in range(4)] + [[c - 1 for c in need]]
    for caps in shorts:
        rc, sz, outs, sts = decode(caps)
        assert rc == abi.GPX_ERANGE and sz == need
        assert all((o == 0xAB).all() for o in outs)
        assert host_bytes(sts) == status.tobytes()
    rc, sz, outs, sts = decode(need)
    assert rc == 0 and sz == need
    assert [host_bytes(o) for o in outs] == [acc.tobytes(), blob.tobytes(), rep.tobytes(), dec.tobytes()]

    L = len(world.lanes)
    for name, recs in (("wire_encode_replies_device", random_replies(rng, world, 300, L)),
                       ("wire_encode_decisions_device", random_decisions(rng, world, 400))):
        host = (wire.encode_replies if "replies" in name else wire.encode_decisions)(e, recs)
        need = [len(host[1]), len(host[2])]
        d = dev_recs(recs, 32)

        def encode(caps):
            out = torch.full((caps[0],), 0xAB, dtype=torch.uint8, device=DEV)
            rf = torch.full((caps[1] * 16,), 0xAB, dtype=torch.uint8, device=DEV)
            rst = torch.full((len(recs),), 0xAB, dtype=torch.uint8, device=DEV)
            nb, nr = C.c_uint64(caps[0]), C.c_uint32(caps[1])
            lead = (C.c_uint32(len(recs)), dptr(d)) if "replies" in name else (dptr(d), None, C.c_uint32(len(recs)))
            rc = cuda_lib.fn(name)(e.handle, *lead, dptr(rst), dptr(out), C.byref(nb), dptr(rf), C.byref(nr), st)
            torch.cuda.synchronize()
            return rc, [nb.value, nr.value], out, rf, rst

        for caps in ([need[0] - 1, need[1]], [need[0], need[1] - 1], [need[0] - 1, need[1] - 1]):
            rc, sz, out, rf, rst = encode(caps)
            assert rc == abi.GPX_ERANGE and sz == need
            assert (out == 0xAB).all() and (rf == 0xAB).all() and host_bytes(rst) == host[0].tobytes()
        rc, sz, out, rf, rst = encode(need)
        assert rc == 0 and sz == need
        assert host_bytes(out) == host[1].tobytes() and host_bytes(rf) == host[2].tobytes()
    e.close()


# ---- two hosts ------------------------------------------------------------------------------------------------------
class DevNode:
    """an engine driven through the device phase calls on torch's current stream"""

    def __init__(self, eng: Engine):
        self.e, self.L = eng, eng.L
        self.st = wire.stream_handle()

    def ctl(self):
        return torch.zeros(8, dtype=torch.int32, device=DEV)  # gpx_dev_ctl

    def accepts(self, d: wire.DecodeOut, ctl, extra):
        na, lanes = d.sizes[0], self.e.n_lanes
        rep = torch.empty((max(na * lanes, 1), 32), dtype=torch.uint8, device=DEV)
        self.L.check(self.L.fn("accepts_device")(self.e.handle, dptr(d.accepts), C.c_uint32(na), dptr(d.blob),
                                                 C.c_uint64(d.sizes[1]), C.c_uint32(0), None, None, dptr(rep),
                                                 dptr(extra), C.c_uint32(extra.shape[0]), dptr(ctl), self.st))
        return rep[: na * lanes]

    def replies(self, rep, n, out_dec, ctl):
        self.L.check(self.L.fn("replies_device")(self.e.handle, dptr(rep), C.c_uint32(n), dptr(out_dec), dptr(ctl),
                                                 self.st))

    def decisions(self, dec, n, extra, ctl):
        ex = torch.zeros((max(n * self.e.n_lanes, 1), 24), dtype=torch.uint8, device=DEV)
        self.L.check(self.L.fn("decisions_device")(self.e.handle, dptr(dec), C.c_uint32(n), dptr(ex), dptr(extra),
                                                   C.c_uint32(extra.shape[0]), dptr(ctl), self.st))
        return ex[: n * self.e.n_lanes]


def ref_nodes(refs):
    return refs.view(torch.int32).reshape(-1, 4)[:, 3]


def exec_and_extra(ex, extra, ctl):
    n_extra = min(int(ctl[2].item()), extra.shape[0])
    return np.concatenate([wire.to_records(ex, abi.exec_dtype), wire.to_records(extra[:n_extra], abi.exec_dtype)])


@pytest.mark.parametrize("R,window", [(3, 8), (5, 1), (3, 1), (5, 8)])
def test_two_hosts_with_records_only_in_hbm_equal_one_oracle_engine(cuda_lib, oracle_lib, R, window):
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
    for r in range(rounds):
        stop = np.zeros(len(gids), bool) if r < rounds - 1 else (gids % 7 == 0)
        reqs, pay = make_requests(gids, payload_len=5 + r, seed=3, round_no=r, entry_lane=0, entry_node=100,
                                  stop_mask=stop)
        acc_a, blob_a, st_a = A.propose(reqs, pay)
        acc_o, blob_o, st_o = O.propose(reqs, pay)
        assert np.array_equal(st_a, st_o) and (st_a > 0).all()
        # A -> B: ACCEPT packets (host codec), one upload
        unnamed = wire.encode_batched_commit("NoSuchGroup", 0, 0, 100, 0, [1], members)
        arena, refs = wire.device_packets(accept_packets(names, 0, acc_a, blob_a) + [unnamed])
        d = wire.decode_batch_device(B, arena, refs, caps.get("acc", (1, 16, 1, 1)))
        caps["acc"] = d.sizes
        assert d.sizes[0] == len(acc_a) and d.sizes[2] == d.sizes[3] == 0
        st = d.status.cpu().numpy()
        assert (st[:-1] == abi.WS_OK).all() and st[-1] == abi.WS_UNKNOWN_NAME
        ctl_b, extra_b = dB.ctl(), torch.zeros((4096, 24), dtype=torch.uint8, device=DEV)
        rep_b = dB.accepts(d, ctl_b, extra_b)
        enc = wire.encode_replies_device(B, rep_b, rep_b.shape[0], caps.get("rep", (64, 1)))
        caps["rep"] = enc.sizes
        assert (ref_nodes(enc.refs) == 100).all()
        assert not (enc.rstatus == abi.WE_NACK).any()
        # B -> A: the reply arena as it is (the decoder ignores the refs' gid and node)
        rep_a, _ = A.handle_accepts(acc_a, blob_a)
        rep_o, _ = O.handle_accepts(acc_o, blob_o)
        ctl_a = dA.ctl()
        dec_a = torch.empty((4 * len(gids), 32), dtype=torch.uint8, device=DEV)  # the tally appends, unbounded
        dA.replies(dev_recs(rep_a, 32), len(rep_a), dec_a, ctl_a)  # its own replies first, as one stable merge by gid
        d2 = wire.decode_batch_device(A, enc.out.clone(), enc.refs.clone(), caps.get("ab", (1, 16, 1, 1)))
        caps["ab"] = d2.sizes
        assert (d2.status == abi.WS_OK).all() and d2.sizes[0] == d2.sizes[3] == 0
        dA.replies(d2.replies, d2.sizes[2], dec_a, ctl_a)
        dec_o = O.handle_accept_replies(rep_o)
        # A -> B: decisions encoded from the tally's device count
        enc2 = wire.encode_decisions_device(A, dec_a, ctl_a.data_ptr() + 4, dec_a.shape[0], caps.get("dec", (64, 1)))
        caps["dec"] = enc2.sizes
        n_dec = int(ctl_a[1].item())
        assert n_dec == len(dec_o) == len(gids)
        assert (enc2.rstatus[:n_dec] == abi.WE_SENT).all() and enc2.sizes[1] == len(gids) * (R - 1)
        sel = ref_nodes(enc2.refs) == 101
        d3 = wire.decode_batch_device(B, enc2.out.clone(), enc2.refs[sel].contiguous(), caps.get("com", (1, 16, 1, 1)))
        caps["com"] = d3.sizes
        assert (d3.status == abi.WS_OK).all() and d3.sizes[3] == len(gids)
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


# ---- PCIe traffic of an acceptor chain ------------------------------------------------------------------------------
def acceptor_packets(G, slot):
    """one ACCEPT per group, 8-byte value, ballot (1, 100) -- above every group's initial ballot -- for node 101"""
    return [wire.encode_accept(wire.Request(f"NoopPaxosApp{i}", 0, slot * G + i, b"12345678", entry_replica=100),
                               slot, 1, 100, False, 0, 100) for i in range(G)]


def chain(node: DevNode, arena, refs, G):
    d = wire.decode_batch_device(node.e, arena, refs, (G, 16 * G, 1, 1))
    ctl, extra = node.ctl(), torch.zeros((1024, 24), dtype=torch.uint8, device=DEV)
    rep = node.accepts(d, ctl, extra)
    return wire.encode_replies_device(node.e, rep, rep.shape[0], (128 * G, G))


def pcie_bytes(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "trace.json")
        prof.export_chrome_trace(p)
        trace = json.load(open(p))
    total, seen = 0, 0
    for ev in trace.get("traceEvents", []):
        name = ev.get("name", "")
        if ev.get("cat") == "gpu_memcpy" and ("HtoD" in name or "DtoH" in name):
            assert "bytes" in ev.get("args", {}), ev
            total += int(ev["args"]["bytes"])
            seen += 1
    return total, seen, out


def test_an_acceptor_chain_moves_no_records_over_pcie(cuda_lib):
    got = {}
    for G in (10_000, 100_000):
        e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=1, lane_node=[101], window=8,
                                         max_batch_recs=G, max_batch_payload=16 * G, log_ring_bytes=1 << 25))
        e.create_groups(group_descs_fast(G, members=(100, 101, 102)))
        wire.set_group_names(e, np.arange(G, dtype=np.uint32), [f"NoopPaxosApp{i}" for i in range(G)])
        node = DevNode(e)
        arena, refs = wire.device_packets(acceptor_packets(G, 0))
        out = chain(node, arena, refs, G)  # warm-up: the scratch grows here
        torch.cuda.synchronize()
        assert out.sizes[1] == G
        arena, refs = wire.device_packets(acceptor_packets(G, 1))  # the caller's upload, outside the chain
        b, seen, out = pcie_bytes(lambda: chain(node, arena, refs, G))
        assert out.sizes[1] == G and (out.rstatus == abi.WE_SENT).all()
        assert seen > 0  # the totals the call reads
        got[G] = b
        e.close()
    assert got[10_000] <= 4096 and got[100_000] <= got[10_000], got
