"""GPU: the response cache through the C ABI (gpx_response_cache_init / _put_device / _match_device).

* The random cases of tests/rc_cases.py -- keys colliding on each field, port 0, expiry exactly at the timeout,
  over-filled buckets, repeated keys, batched requests, gids named again or unnamed between put and match -- give the
  model's hit[], misses and miss count, with and without name state.
* End to end on one engine hosting all three replicas: client REQUEST packets (fresh requests, retransmissions of
  requests executed in earlier rounds, some of them after their entries expired, and batched RequestPackets) go through
  gpx_wire_decode_requests_device -- or, as JSON REQUEST members of BATCHED_PAXOS_PACKETs, gpx_wire_decode_json_device
  and gpx_wire_decode_json_requests_device -- then match, then the device round; the executed requests' keys are put
  from the EXEC records.  The EXEC records (but for their log-ring positions), statuses and rows equal a second
  engine's that is given only the model's misses, and no request the model answers is executed again.
* Error paths: GPX_EINVAL before init, for a bad n_buckets and for a negative handle or a gid >= max_groups, with
  nothing written.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import Engine, abi, group_descs, make_config
from rc_cases import Cache, Names, random_case
from test_wire_coord_gpu import request_arena
from test_wire_device_gpu import dev_recs
from wire_coord_cases import NOW_MS
from wire_fwd_cases import wrapper

from gigapaxos_b200 import packets_json as pj
from gigapaxos_b200 import wire

pytestmark = pytest.mark.gpu

DEV = "cuda"
EINVAL = "gpx error %d:" % abi.GPX_EINVAL
NAMES = lambda gids: [f"NoopPaxosApp{int(g)}" for g in gids]


def dev(a: np.ndarray):
    return dev_recs(a, a.dtype.itemsize) if len(a) else torch.zeros((1, a.dtype.itemsize), dtype=torch.uint8,
                                                                     device=DEV)


def match(e, reqs, meta, now, d_reqs=None, d_meta=None, n=None):
    """-> (hit, out_reqs, out_meta) as numpy"""
    n = len(reqs) if n is None else n
    d_reqs = dev(reqs) if d_reqs is None else d_reqs
    d_meta = dev(meta) if d_meta is None else d_meta
    hit = torch.full((max(n, 1),), 0x55, dtype=torch.int32, device=DEV)
    out_r = torch.zeros((max(n, 1), 32), dtype=torch.uint8, device=DEV)
    out_m = torch.zeros((max(n, 1), 32), dtype=torch.uint8, device=DEV)
    k = e.response_cache_match(d_reqs, d_meta, n, now, hit, out_r, out_m)
    torch.cuda.synchronize()
    return (hit[:n].cpu().numpy(), wire.to_records(out_r[:k], abi.request_dtype),
            wire.to_records(out_m[:k], abi.req_meta_dtype))


def put(e, keys, now):
    e.response_cache_put(dev(keys), len(keys), now)
    torch.cuda.synchronize()


@pytest.mark.parametrize("names_on", [True, False])
def test_c_abi_gives_the_models_matches(cuda_lib, names_on):
    G = 8
    seen = hits = 0
    for seed in range(30):
        n_buckets, T, _, ops = random_case(np.random.default_rng(seed + (0 if names_on else 500)), G=G)
        e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=3, lane_node=[100, 101, 102]))
        descs = group_descs(G)
        e.create_groups(descs)
        e.response_cache_init(n_buckets, T)
        names = Names(G, on=names_on)
        model = Cache(n_buckets, T, names)
        if names_on:  # every gid named once; without name state every gid counts as named at generation 0
            names.name(range(G))
            wire.set_group_names(e, np.arange(G), NAMES(range(G)))
        for op in ops:
            if op[0] == "name" and names_on:
                names.name(op[1])
                wire.set_group_names(e, op[1], NAMES(op[1]))
            elif op[0] == "drop" and names_on:
                names.drop(op[1])
                e.destroy_groups(op[1])
                e.create_groups(descs[op[1]])
            elif op[0] == "put":
                assert model.put(op[1], op[2]) == 0
                put(e, op[1], op[2])
            elif op[0] == "match":
                _, reqs, meta, now = op
                hit, out_r, out_m = match(e, reqs, meta, now)
                want, miss = model.match(reqs, meta, now)
                assert hit.tolist() == want.tolist()
                assert out_r.tobytes() == reqs[miss].tobytes() and out_m.tobytes() == meta[miss].tobytes()
                seen += len(reqs)
                hits += int((want >= 0).sum())
        e.close()
    assert seen > 0 and hits > 0


# ---- end to end ---------------------------------------------------------------------------------------------------
class Client:
    """the requests of a run: fresh ones, retransmissions of executed ones (the same RequestPacket again) and batched
    RequestPackets"""

    def __init__(self, G, rng):
        self.G, self.rng, self.next_id = G, rng, 1 << 20
        self.executed = []  # Requests executed in earlier rounds

    def fresh(self, gid):
        self.next_id += 1
        port = int(self.rng.choice([0, 4567, 4568]))
        return wire.Request(NAMES([gid])[0], 0, self.next_id, bytes(self.rng.integers(65, 91, size=5, dtype=np.uint8)),
                            client=("10.1.2.3", port) if port else None)

    def packets(self):
        out = [self.fresh(int(g)) for g in self.rng.choice(self.G, size=self.G // 2, replace=False)]
        if self.executed:
            k = min(len(self.executed), self.G // 4)
            out += [self.executed[int(i)] for i in self.rng.choice(len(self.executed), size=k, replace=False)]
        for g in self.rng.choice(self.G, size=4, replace=False):  # batched: never a hit, whatever the cache holds
            outer = self.executed[int(self.rng.integers(len(self.executed)))] if self.executed else self.fresh(int(g))
            out.append(wire.Request(outer.paxos_id, 0, outer.request_id, outer.value, client=outer.client,
                                    batched=(self.fresh(int(outer.paxos_id[len("NoopPaxosApp"):])),)))
        return [out[int(i)] for i in self.rng.permutation(len(out))]


def decode(e, pkts, form):
    """client packets received at node 100 -> (reqs, meta, payload) device tensors, n, payload bytes"""
    if form == "bytes":
        arena, refs = request_arena([(wire.encode_request(r), 100) for r in pkts])
        d = wire.decode_requests_device(e, arena, refs, NOW_MS, (1, 16))
    else:
        wraps, i = [], 0
        while i < len(pkts):
            k = int(1 + i % 5)
            wraps.append(wrapper([pj.request_json(r) for r in pkts[i: i + k]]))
            i += k
        arena, refs = request_arena([(w, 100) for w in wraps])
        j = wire.decode_json_device(e, arena, refs, (1, 1, 1))
        d = wire.decode_json_requests_device(e, arena, refs, j.members, j.sizes[0], NOW_MS, (1, 16))
    torch.cuda.synchronize()
    if form == "bytes":
        assert (d.status == abi.WS_OK).all()
    return d.reqs, d.meta, d.payload, d.sizes[0], d.sizes[1]


def device_round(e, d_reqs, n, d_pay, pay_bytes):
    L = e.n_lanes
    st = torch.zeros(max(n, 1), dtype=torch.int32, device=DEV)
    ex = torch.zeros((max(n * L, 1), 24), dtype=torch.uint8, device=DEV)
    bufs = abi.DevRoundBufs(d_reqs.data_ptr(), d_pay.data_ptr(), pay_bytes, n, st.data_ptr(), ex.data_ptr())
    e.L.check(e.L.fn("round_device")(e.handle, C.byref(bufs), wire.stream_handle()))
    torch.cuda.synchronize()
    return st[:n].cpu().numpy(), wire.to_records(ex[: n * L], abi.exec_dtype)


def same_exec(a, b):
    """the same EXEC records but for payload_off, a position in the lane's log ring: where a slot that carries several
    requests gets its constructed blob is left to the order the round's threads reserve space in"""
    a, b = a.copy(), b.copy()
    a["payload_off"] = b["payload_off"] = 0
    return a.tobytes() == b.tobytes()


@pytest.mark.parametrize("form", ["bytes", "json"])
def test_retransmissions_are_answered_and_not_executed_again(cuda_lib, form):
    G, T = 256, 10_000
    cfg = dict(max_groups=G, n_lanes=3, lane_node=[100, 101, 102], max_batch_recs=4 * G)
    A = Engine(cuda_lib, make_config(cuda_lib, **cfg))
    B = Engine(cuda_lib, make_config(cuda_lib, **cfg))
    for e in (A, B):
        e.create_groups(group_descs(G))
    gids = np.arange(G, dtype=np.uint32)
    wire.set_group_names(A, gids, NAMES(gids))
    A.response_cache_init(1 << 10, T)
    names = Names(G)
    names.name(range(G))
    model = Cache(1 << 10, T, names)
    rng = np.random.default_rng(17 if form == "bytes" else 18)
    client = Client(G, rng)
    handle, total_hits, re_executed = 0, 0, 0
    for r in range(8):
        now = NOW_MS + 3000 * r  # entries of round r expire in round r + 4
        pkts = client.packets()
        d_reqs, d_meta, d_pay, n, pay_bytes = decode(A, pkts, form)
        reqs, meta = wire.to_records(d_reqs[:n], abi.request_dtype), wire.to_records(d_meta[:n], abi.req_meta_dtype)
        want, miss = model.match(reqs, meta, now)
        hit, out_r, out_m = match(A, reqs, meta, now, d_reqs, d_meta, n)
        assert hit.tolist() == want.tolist()
        assert out_r.tobytes() == reqs[miss].tobytes() and out_m.tobytes() == meta[miss].tobytes()
        total_hits += int((want >= 0).sum())
        # the round: A proposes the misses match left in its output, B the model's misses
        k = len(miss)
        d_out = dev(out_r)
        st_a, ex_a = device_round(A, d_out, k, d_pay, pay_bytes)
        st_b, ex_b = device_round(B, dev(reqs[miss]), k, d_pay.clone(), pay_bytes)
        assert st_a.tolist() == st_b.tolist() and same_exec(ex_a, ex_b)
        executed = set()
        for x in ex_a[(ex_a["flags"] & abi.F_VOID) == 0]:
            executed.add((int(x["gid"]), int(x["req_id"])))
        missed = {(int(q["gid"]), int(q["req_id"])) for q in reqs[miss]}
        for q in reqs[want >= 0]:
            key = (int(q["gid"]), int(q["req_id"]))
            assert key not in executed or key in missed
        # put the executed requests' keys, in request order, as a node's app does after Replicable.execute
        keys = []
        for q, m in zip(reqs[miss], meta[miss]):
            if (int(q["gid"]), int(q["req_id"])) not in executed:
                continue
            kk = np.zeros(1, abi.rc_key_dtype)
            kk["gid"], kk["req_id"], kk["handle"] = q["gid"], q["req_id"], handle
            kk["client_ip"], kk["client_port"] = m["client_ip"], m["client_port"]
            keys.append(kk)
            handle += 1
        keys = np.concatenate(keys) if keys else np.zeros(0, abi.rc_key_dtype)
        assert model.put(keys, now) == 0
        put(A, keys, now)
        done = {p.request_id for p in client.executed}
        re_executed += sum(1 for q in reqs[miss] if (int(q["gid"]), int(q["req_id"])) in executed
                           and int(q["req_id"]) in done)
        by_id = {}
        for p in pkts:
            for x in (p,) + tuple(p.batched):
                by_id[x.request_id] = x
        client.executed += [by_id[int(q["req_id"])] for q in reqs[miss]
                            if (int(q["gid"]), int(q["req_id"])) in executed and int(q["req_id"]) in by_id
                            and not by_id[int(q["req_id"])].batched]
    for lane in range(3):
        assert A.dump_rows(gids, lane).tobytes() == B.dump_rows(gids, lane).tobytes()
    assert total_hits > G // 4 and re_executed > 0  # answered retransmissions, and expired or batched ones executed
    for e in (A, B):
        e.close()


def test_error_paths_write_nothing(cuda_lib):
    G = 8
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=3, lane_node=[100, 101, 102]))
    e.create_groups(group_descs(G))
    k = np.zeros(2, abi.rc_key_dtype)
    k["gid"], k["req_id"], k["handle"] = [1, 2], [5, 6], [10, 11]
    r = np.zeros(2, abi.request_dtype)
    r["gid"], r["req_id"], r["client"] = [1, 2], [5, 6], [0, 1]
    m = np.zeros(2, abi.req_meta_dtype)
    hit = torch.zeros(2, dtype=torch.int32, device=DEV)
    o = torch.zeros((2, 32), dtype=torch.uint8, device=DEV)
    with pytest.raises(abi.GpxError, match=EINVAL):
        e.response_cache_put(dev(k), 2, 0)
    with pytest.raises(abi.GpxError, match=EINVAL):
        e.response_cache_match(dev(r), dev(m), 2, 0, hit, o, o.clone())
    for nb in (0, 3, 1 << 25, 0xFFFFFFFF):
        with pytest.raises(abi.GpxError, match=EINVAL):
            e.response_cache_init(nb, 100)
    with pytest.raises(abi.GpxError, match=EINVAL):
        e.response_cache_init(16, -1)
    e.response_cache_init(1, 100)
    put(e, k[:1], 0)
    for bad in ("handle", "gid"):
        kb = k.copy()
        kb[1][bad] = -1 if bad == "handle" else G
        with pytest.raises(abi.GpxError, match=EINVAL):
            e.response_cache_put(dev(kb), 2, 0)
    # nothing written: key 0 still answers, key 1 does not
    assert match(e, r, m, 1)[0].tolist() == [10, -1]
    e.response_cache_init(1, 100)  # again: cleared
    assert match(e, r, m, 1)[0].tolist() == [-1, -1]
    e.close()
