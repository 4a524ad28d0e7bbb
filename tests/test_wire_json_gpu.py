"""GPU: gpx_wire_decode_json_device through the C ABI.

* Scale: 100 K groups; the same logical BatchedAcceptReplies and BatchedCommits as bytes (gpx_wire_decode_batch_device)
  and as JSON -- 4 MiB BATCHED_PAXOS_PACKET wrappers mixed with thousands of bare packets -- give identical records; each
  member's status is its byte packet's, and the member table is the splitter's spans.
* The malformed corpus and singleton ACCEPT_REPLYs of tests/wire_json_cases.py against its schema model.
* GPX_ERANGE with an output one short: the sizes are reported and every output is left as it was.
* Streams: the call on a side stream between byte decodes on torch's default stream, all sharing the wire scratch.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import abi
from test_wire_dev_gpu import world_engine
from wire_dev_cases import World, random_world
from wire_json_cases import as_bytes, as_json, malformed_corpus, model_batch, random_logical, wrap

from gigapaxos_b200 import packets_json as pj, wire

pytestmark = pytest.mark.gpu

MIB4 = 4 << 20


def fast_world(rng, G):
    pool = [98, 99, 100, 101, 102, 103, 104]
    groups = {}
    for gid in range(G):
        R = int(rng.integers(1, 6))
        groups[gid] = ("grp/%dé" % gid, int(rng.integers(0, 3)), sorted(int(x) for x in rng.choice(pool, R, replace=False)))
    return World(groups)


def pack_mixed(rng, js):
    """JSON members -> (packets, spans, order): wrappers of up to 4 MiB, every fifth member a bare packet; order[j] is
    the index in js of the j-th member in packet order (a bare packet overtakes the wrapper still being filled)"""
    pkts, spans, order, cur = [], [], [], []

    def flush():
        if cur:
            w, sp = wrap([js[i] for i in cur])
            pkts.append(w)
            spans.extend((len(pkts) - 1, o, l) for o, l in sp)
            order.extend(cur)
            cur.clear()
    size = 0
    for i, m in enumerate(js):
        if i % 5 == 4:
            pkts.append(m)
            spans.append((len(pkts) - 1, 0, len(m)))
            order.append(i)
            continue
        if size + len(m) + 64 > MIB4:
            flush()
            size = 0
        cur.append(i)
        size += len(m) + 1
    flush()
    return pkts, spans, order


def decode_json(e, pkts, nodes=None, caps=(0, 0, 0), stream=None):
    arena, refs = wire.pack_packets(pkts)
    if nodes is not None:
        refs["node"] = nodes
    import torch
    da = torch.from_numpy(arena.copy()).cuda()
    dr = torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16)).cuda()
    out = wire.decode_json_device(e, da, dr, caps, stream)
    return (out.status.cpu().numpy(), wire.to_records(out.members, abi.wire_member_dtype),
            wire.to_records(out.replies, abi.reply_dtype), wire.to_records(out.decisions, abi.decision_dtype), refs)


def test_json_decode_equals_the_byte_decode_at_100k_groups(cuda_lib):
    rng = np.random.default_rng(1)
    world = fast_world(rng, 100_000)
    e = world_engine(cuda_lib, world)
    logical = random_logical(rng, world, 70_000)
    js = [as_json(k, f) for k, f in logical]
    pkts, spans, order = pack_mixed(rng, js)
    byts = [as_bytes(*logical[i]) for i in order]  # the byte packets in the JSON members' order
    bst, _, _, brep, bdec = wire.decode_batch(e, byts)
    assert max(len(p) for p in pkts) > MIB4 - 4096 and sum(len(p) < 4096 for p in pkts) > 10_000
    st, mem, rep, dec, refs = decode_json(e, pkts)
    assert (st == abi.WS_OK).all()
    assert [(int(m["pkt"]), int(m["off"]) - int(refs["off"][m["pkt"]]), int(m["len"])) for m in mem] == spans
    assert np.array_equal(mem["status"], bst)
    assert np.array_equal(rep, brep) and np.array_equal(dec, bdec) and len(rep) > 10_000
    e.close()


def test_malformed_corpus_and_singletons_match_the_schema_model(cuda_lib):
    world = random_world(np.random.default_rng(9), 30)
    e = world_engine(cuda_lib, world)
    cases = malformed_corpus(world)
    rng = np.random.default_rng(4)
    for gid, (name, ver, members) in list(world.groups.items())[:10]:
        for node in (100, 101, 98):
            cases.append((pj.accept_reply_json(name, ver, members[0], 7, 103, 11, 10, int(rng.integers(-2**40, 2**40)),
                                               undigest_request=bool(rng.integers(0, 4) == 0)), node))
    pkts, nodes = [p for p, _ in cases], [n for _, n in cases]
    st, mem, rep, dec, _ = decode_json(e, pkts, nodes)
    est, ems, erep, edec = model_batch(world, pkts, nodes)
    assert list(st) == est and list(mem["status"]) == ems
    assert np.array_equal(rep, erep) and np.array_equal(dec, edec)
    e.close()


def test_output_one_short_reports_sizes_and_writes_nothing(cuda_lib):
    import torch
    rng = np.random.default_rng(2)
    world = random_world(rng, 40)
    e = world_engine(cuda_lib, world)
    js = [as_json(k, f) for k, f in random_logical(rng, world, 300)]
    pkts, _, _ = pack_mixed(rng, js)
    st, mem, rep, dec, _ = decode_json(e, pkts)
    full = (len(mem), len(rep), len(dec))
    arena, refs = wire.pack_packets(pkts)
    da = torch.from_numpy(arena.copy()).cuda()
    dr = torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16)).cuda()
    for short in range(3):
        caps = [c - (j == short) for j, c in enumerate(full)]
        bufs = [torch.full((max(c, 1) * w,), 0xAB, dtype=torch.uint8, device="cuda") for c, w in zip(caps, (16, 32, 32))]
        status = torch.full((len(pkts),), 0x55, dtype=torch.int32, device="cuda")
        sz = [C.c_uint32(c) for c in caps]
        rc = e.L.fn("wire_decode_json_device")(e.handle, C.c_uint32(len(pkts)), C.c_void_p(da.data_ptr()),
                                               C.c_uint64(da.numel()), C.c_void_p(dr.data_ptr()),
                                               C.c_void_p(status.data_ptr()), C.c_void_p(bufs[0].data_ptr()),
                                               C.byref(sz[0]), C.c_void_p(bufs[1].data_ptr()), C.byref(sz[1]),
                                               C.c_void_p(bufs[2].data_ptr()), C.byref(sz[2]), wire.stream_handle())
        assert rc == abi.GPX_ERANGE
        assert tuple(s.value for s in sz) == full
        torch.cuda.synchronize()
        assert all(bool((b == 0xAB).all()) for b in bufs)
    e.close()


def test_runs_on_a_side_stream_between_byte_decodes(cuda_lib):
    import torch
    rng = np.random.default_rng(5)
    world = random_world(rng, 50)
    e = world_engine(cuda_lib, world)
    logical = random_logical(rng, world, 3000)
    pkts, _, order = pack_mixed(rng, [as_json(k, f) for k, f in logical])
    byts = [as_bytes(*logical[i]) for i in order]
    bst, _, _, brep, bdec = wire.decode_batch(e, byts)
    ba, br = wire.device_packets(byts)
    arena, refs = wire.pack_packets(pkts)
    ja = torch.from_numpy(arena.copy()).cuda()
    jr = torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16)).cuda()
    side = torch.cuda.Stream()
    for _ in range(3):
        b1 = wire.decode_batch_device(e, ba, br, (0, 0, 0, 0))
        side.wait_stream(torch.cuda.current_stream())
        j = wire.decode_json_device(e, ja, jr, (0, 0, 0), stream=side)
        torch.cuda.current_stream().wait_stream(side)
        b2 = wire.decode_batch_device(e, ba, br, (0, 0, 0, 0))
        for b in (b1, b2):
            assert np.array_equal(wire.to_records(b.replies, abi.reply_dtype), brep)
        assert np.array_equal(wire.to_records(j.replies, abi.reply_dtype), brep)
        assert np.array_equal(wire.to_records(j.decisions, abi.decision_dtype), bdec)
        assert np.array_equal(wire.to_records(j.members, abi.wire_member_dtype)["status"], bst)
    e.close()
