"""GPU: a client's own REQUEST packets through the C ABI (gpx_wire_decode_client_requests_device).

* Random client traffic and the one-rule-per-case corpus of tests/wire_client_cases.py give the model's statuses,
  requests, meta and payload byte for byte, with and without peers.
* At 100 K and 1 M client packets of one small request each, every output equals
  gpx_wire_decode_json_requests_device's over the same requests with the resolved "CA" / "LA" written out.
* End to end at a coordinator (node 100, its peers remote): decode, put the executed requests' keys into the response
  cache, decode a retransmission from the same connection (a hit) and the same request ids from another client port
  (misses), propose the misses with gpx_propose_device_heads and encode their ACCEPTs with
  gpx_wire_encode_accepts_device: the bytes are gpx_wire_encode_accept's, with the connection's client address."""
import numpy as np
import pytest
import torch

from helpers import Engine, abi, group_descs, make_config
from test_wire_coord_gpu import request_arena
from test_wire_dev_gpu import world_engine
from test_wire_device_gpu import dev_recs, host_bytes
from wire_client_cases import bulk_client_packets, corpus, expected, peer_rows, random_client_packets
from wire_coord_cases import NOW_MS, expected_accepts
from wire_dev_cases import World, random_world

from gigapaxos_b200 import packets_json as pj
from gigapaxos_b200 import wire
from gigapaxos_b200.spread import coordinator_of

pytestmark = pytest.mark.gpu

DEV = "cuda"


def decode(e, pkts, peers, caps=(1, 16)):
    arena, refs = request_arena(pkts)
    pr = None if peers is None else dev_recs(peer_rows(peers), 16)
    d = wire.decode_client_requests_device(e, arena, refs, pr, NOW_MS, caps)
    torch.cuda.synchronize()
    return d


def as_numpy(d):
    return (d.status.cpu().numpy(), wire.to_records(d.reqs, abi.request_dtype), wire.to_records(d.meta, abi.req_meta_dtype),
            d.payload.cpu().numpy())


def assert_model(got, want):
    st, reqs, meta, pay = got
    est, ereqs, emeta, epay = want
    assert st.tolist() == est.tolist()
    assert reqs.tobytes() == ereqs.tobytes() and meta.tobytes() == emeta.tobytes() and pay.tobytes() == epay.tobytes()


@pytest.mark.parametrize("seed", [1, 2])
def test_client_packets_give_the_models_outputs(cuda_lib, seed):
    rng = np.random.default_rng(seed)
    world = random_world(rng, 60)
    e = world_engine(cuda_lib, world)
    pkts, peers = random_client_packets(rng, world, 2000)
    for given in (True, False):
        assert_model(as_numpy(decode(e, pkts, peers if given else None)), expected(world, pkts, peers if given else None))
    cases = corpus(world)
    for with_peers in (True, False):
        sel = [c for c in cases if (c[2] is not None) == with_peers]
        got = as_numpy(decode(e, [(c[0], c[1]) for c in sel], [c[2] for c in sel] if with_peers else None))
        assert got[0].tolist() == [c[3] for c in sel]
        assert_model(got, expected(world, [(c[0], c[1]) for c in sel], [c[2] for c in sel] if with_peers else None))
    e.close()


def arena_members(pkts, node):
    arena, refs = request_arena([(b, node) for b in pkts])
    r = wire.to_records(refs, abi.wire_ref_dtype)
    mem = np.zeros(len(r), abi.wire_member_dtype)
    mem["pkt"], mem["off"], mem["len"], mem["status"] = np.arange(len(r)), r["off"], r["len"], abi.WS_UNHANDLED
    return arena, refs, dev_recs(mem, 16)


@pytest.mark.parametrize("n", [100_000, 1_000_000])
def test_equals_the_json_requests_decoder_with_the_addresses_written_out(cuda_lib, n):
    G = 4096
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=3, lane_node=[100, 101, 102]))
    e.create_groups(group_descs(G))
    wire.set_group_names(e, np.arange(G), [f"NoopPaxosApp{g}" for g in range(G)])
    plain, inserted, peers = bulk_client_packets(n, G, np.random.default_rng(n))
    arena, refs, _ = arena_members(plain, 100)
    got = wire.decode_client_requests_device(e, arena, refs, dev_recs(peers, 16), NOW_MS, (n, 16 * n))
    ia, ir, mem = arena_members(inserted, 100)
    want = wire.decode_json_requests_device(e, ia, ir, mem, n, NOW_MS, (n, 16 * n))
    torch.cuda.synchronize()
    assert got.sizes == want.sizes and got.sizes[0] == n
    assert (got.status == abi.WS_OK).all() and torch.equal(got.status, want.status)
    for a, b in ((got.reqs, want.reqs), (got.meta, want.meta), (got.payload, want.payload)):
        assert torch.equal(a, b)
    meta = wire.to_records(got.meta[:1000], abi.req_meta_dtype)
    assert (meta["client_port"] >= 1024).all() and (meta["listen_port"] == 2000).all()
    e.close()


def test_retransmission_from_the_same_connection_is_answered_from_the_cache(cuda_lib):
    R, G = 3, 64
    members = [100, 101, 102]
    names = [f"NoopPaxosApp{g}" for g in range(G)]
    coord = np.array([coordinator_of(s, members) for s in names])
    gids = [int(g) for g in np.nonzero(coord == 100)[0]]
    world = World({g: (names[g], 0, members) for g in gids}, lanes=[100])
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, n_lanes=1, lane_node=[100], max_group_size=R,
                                     max_batch_recs=4 * G))
    e.create_groups(group_descs(G))
    wire.set_group_names(e, gids, [names[g] for g in gids])
    e.response_cache_init(1 << 10, 60_000)
    conn, other, lis = ("10.1.2.3", 40001), ("10.1.2.3", 40002), ("10.0.0.9", 2000)
    reqs_in = [wire.Request(names[g], 0, 1000 + k, b"op%d" % k, entry_time=5) for k, g in enumerate(gids)]
    pkts = [(pj.client_request_json(r), 100) for r in reqs_in]
    d = decode(e, pkts, [(conn, lis)] * len(pkts))
    st, reqs, meta, _ = as_numpy(d)
    assert (st == abi.WS_OK).all() and len(reqs) == len(gids)
    assert {(tuple(m["client_ip"]), int(m["client_port"])) for m in meta} == {((10, 1, 2, 3), 40001)}
    # executed: their keys go into the cache
    keys = np.zeros(len(reqs), abi.rc_key_dtype)
    keys["gid"], keys["req_id"], keys["handle"] = reqs["gid"], reqs["req_id"], np.arange(len(reqs))
    keys["client_ip"], keys["client_port"] = meta["client_ip"], meta["client_port"]
    e.response_cache_put(dev_recs(keys, 24), len(keys), NOW_MS)
    # the client retransmits one request over the same connection, another client sends the same ids from its port
    again = [pkts[0], pkts[1]]
    d2 = decode(e, again + again, [(conn, lis)] * 2 + [(other, lis)] * 2)
    n2 = d2.sizes[0]
    hit = torch.full((n2,), 0x55, dtype=torch.int32, device=DEV)
    out_r = torch.zeros((n2, 32), dtype=torch.uint8, device=DEV)
    out_m = torch.zeros((n2, 32), dtype=torch.uint8, device=DEV)
    k = e.response_cache_match(d2.reqs, d2.meta, n2, NOW_MS + 10, hit, out_r, out_m)
    torch.cuda.synchronize()
    r2 = wire.to_records(d2.reqs, abi.request_dtype)
    by_client = {int(q["client"]): h for q, h in zip(r2, hit.cpu().tolist())}
    assert sorted(by_client[c] for c in (0, 1)) == [0, 1]  # answered from the cache: the handles put above
    assert by_client[2] == by_client[3] == -1 and k == 2  # another client port: a different request
    # the misses are proposed and their ACCEPTs encoded; they carry the other client's connection
    st_p = torch.empty(k, dtype=torch.int32, device=DEV)
    acc = torch.empty((k, 48), dtype=torch.uint8, device=DEV)
    heads = torch.empty(k, dtype=torch.int32, device=DEV)
    ctl = torch.zeros(8, dtype=torch.int32, device=DEV)
    wire.propose_device_heads(e, out_r, k, d2.payload, d2.sizes[1], st_p, acc, heads, ctl)
    ea = wire.encode_accepts_device(e, acc, ctl.data_ptr(), k, heads, out_r, out_m, k, d2.payload, (1, 1))
    torch.cuda.synchronize()
    na = int(ctl[0].item())
    assert na == 2
    acc_h = wire.to_records(acc[:na], abi.accept_dtype)
    heads_h = heads[:na].cpu().numpy().view(np.uint32)
    rq, mt = wire.to_records(out_r[:k], abi.request_dtype), wire.to_records(out_m[:k], abi.req_meta_dtype)
    est, exp = expected_accepts(world, set(gids), acc_h, heads_h, rq, mt, d2.payload.cpu().numpy(), count=na)
    assert host_bytes(ea.rstatus[:na]) == est.tobytes() and (est == abi.WE_SENT).all()
    got = wire.unpack_packets(ea.out.cpu().numpy(), wire.to_records(ea.refs, abi.wire_ref_dtype))
    assert got == exp and len(got) == 2 * (R - 1)
    assert {(int(m["client_port"]), int(m["listen_port"])) for m in mt} == {(40002, 2000)}
    e.close()
