"""Cases and expectations shared by tests/test_wire_coord.py (the coordinator's wire kernels on the host,
tests/emu/wire_emu.cpp) and tests/test_wire_coord_gpu.py (the same kernels through the C ABI): REQUEST packets
made by the host codec and what decoding them must give, and ACCEPT records with their requests and the AcceptPacket
bytes gpx_wire_encode_accept writes for them."""
from __future__ import annotations

import numpy as np

from gigapaxos_b200 import abi, wire
from wire_dev_cases import World, i32, wrap32
from wrap_cases import BALLOT_BASE, SLOT_BASES

NOW_MS = 1_700_000_000_123
ADDRS = [None, ("10.0.0.1", 2000), ("192.168.7.9", 65535), ("0.0.0.0", 1)]


def random_request(rng, name, version, batched=0, host_only=False):
    """a RequestPacket with every address and flag combination; entryReplica unset (-1) about a third of the time;
    host_only: a digest or a responseValue"""
    val = bytes(rng.integers(0, 256, size=int(rng.integers(0, 40))).astype(np.uint8))
    subs = tuple(random_request(rng, name, version) for _ in range(batched))
    entry = int(rng.choice([-1, -1, 100, 101, 102, 7]))
    digest, response = None, b""
    if host_only:
        if rng.integers(0, 2):
            digest = b"d" * int(rng.integers(1, 5))
        else:
            response = b"r" * int(rng.integers(1, 5))
    return wire.Request(name, version, int(rng.integers(-(1 << 62), 1 << 62)), val, stop=bool(rng.integers(0, 4) == 0),
                        entry_replica=entry, entry_time=int(rng.integers(0, 1 << 41)),
                        client=ADDRS[int(rng.integers(0, len(ADDRS)))], listen=ADDRS[int(rng.integers(0, len(ADDRS)))],
                        should_return=bool(rng.integers(0, 2)), forward_count=int(rng.integers(0, 4)),
                        broadcasted=bool(rng.integers(0, 2)), digest=digest, response=response, batched=subs)


def random_request_packets(rng, world: World, n):
    """[(bytes, receiving node, Request or None)]: singles, batched with 1-20 latched requests, unknown names, stale
    versions, digests and responses, and receiving nodes that are not local or not members"""
    out = []
    gids = list(world.groups)
    for _ in range(n):
        gid = int(rng.choice(gids))
        name, ver, members = world.groups[gid]
        u = int(rng.integers(0, 25))
        if u == 0:
            name = name[:-1] + ("?" if name[-1] != "?" else "!")
        elif u == 1:
            ver = ver + 1
        nb = 0 if rng.integers(0, 2) else int(rng.integers(1, 21))
        host_only = u == 2
        req = random_request(rng, name, ver, batched=nb)
        if host_only:  # in the outer request or in a latched one
            tgt = req if not req.batched or rng.integers(0, 2) else req.batched[int(rng.integers(0, len(req.batched)))]
            if rng.integers(0, 2):
                tgt.digest = b"dd"
            else:
                tgt.response = b"resp"
        local = [m for m in members if m in world.lanes]
        node = int(rng.choice(local)) if local and rng.integers(0, 6) else int(rng.choice(world.lanes + [7]))
        out.append((wire.encode_request(req), node, req))
    return out


def malformed_request_packets(world: World):
    """[(bytes, node, expected status)]"""
    gid = min(g for g in world.groups if any(m in world.lanes for m in world.groups[g][2]))
    name, ver, members = world.groups[gid]
    node = next(m for m in members if m in world.lanes)
    good = wire.encode_request(wire.Request(name, ver, 5, b"xy", entry_replica=node))
    inner = wire.Request(name, ver, 6, b"z", batched=(wire.Request(name, ver, 7, b"w"),))
    nested = wire.encode_request(wire.Request(name, ver, 8, b"q", batched=(inner,)))
    acc = wire.encode_accept(wire.Request(name, ver, 5, b"xy"), 1, 0, node, False, 0, node)
    return [
        (good[:-1], node, abi.WS_MALFORMED),                                # truncated
        (good + b"\0", node, abi.WS_MALFORMED),                             # trailing bytes
        (good[:-4] + b"\xff\xff\xff\xff", node, abi.WS_MALFORMED),          # negative n_batched
        (nested, node, abi.WS_MALFORMED),                                   # a latched request with latched requests
        (b"\0\0\0\x5b" + good[4:], node, abi.WS_MALFORMED),                 # magic 91
        (b"", node, abi.WS_MALFORMED),
        (b'{"type":1}', node, abi.WS_UNHANDLED),                            # JSON
        (acc, node, abi.WS_UNHANDLED),                                      # an ACCEPT is not a REQUEST
        (good, 7, abi.WS_NOT_LOCAL),                                        # no lane serves node 7
        (good, node, abi.WS_OK),
    ]


def expected_requests(world: World, pkts):
    """(status, reqs, meta, values) the request decoder must give for [(bytes, node, Request or None)]"""
    status, rows = [], []
    for k, (b, node, req) in enumerate(pkts):
        if req is None:
            status.append(None)
            continue
        reqs = [req] + list(req.batched)
        if any(r.digest or r.response for r in reqs):
            status.append(abi.WS_UNHANDLED)
            continue
        gid = world.by_name.get(req.paxos_id)
        if gid is None:
            status.append(abi.WS_UNKNOWN_NAME)
            continue
        if world.groups[gid][1] != req.version:
            status.append(abi.WS_VERSION)
            continue
        lane = world.lane_of(node)
        if lane is None or node not in world.groups[gid][2]:
            status.append(abi.WS_NOT_LOCAL)
            continue
        status.append(abi.WS_OK)
        for r in reqs:
            rec = np.zeros(1, abi.request_dtype)[0]
            rec["gid"], rec["flags"], rec["req_id"] = gid, (abi.F_STOP if r.stop else 0) | (lane << 8), r.request_id
            rec["payload_len"], rec["client"] = len(r.value), k
            m = wire.req_meta(r)
            if r.entry_replica == -1:
                rec["entry_node"], m["entry_time"] = node, NOW_MS
            else:
                rec["entry_node"] = r.entry_replica
            rows.append((gid, rec, m, r.value))
    rows.sort(key=lambda t: t[0])  # stable: packet order, then request order, within a gid
    return (status, np.array([t[1] for t in rows], abi.request_dtype), np.array([t[2] for t in rows], abi.req_meta_dtype),
            [t[3] for t in rows])


def check_requests(world, pkts, got):
    """got = (status, reqs, meta, payload) of a device (or emulated) decode"""
    status, reqs, meta, payload = got
    est, ereqs, emeta, vals = expected_requests(world, pkts)
    assert [int(s) for s, e in zip(status, est) if e is not None] == [e for e in est if e is not None]
    assert len(reqs) == len(ereqs)
    for r, v in zip(reqs, vals):
        off = int(r["payload_off"])
        assert off % 16 == 0 and bytes(payload[off: off + len(v)]) == v
    for f in abi.request_dtype.names:
        if f != "payload_off":
            assert np.array_equal(reqs[f], ereqs[f]), f
    assert meta.tobytes() == emeta.tobytes()


# ---- ACCEPTs -> AcceptPacket bytes ------------------------------------------------------------------------------------
def to_request(world: World, reqs, meta, payload, q, batched=()):
    """the wire.Request that reqs[q] / meta[q] stand for"""
    r, m = reqs[q], meta[q]
    name, ver, _ = world.groups[int(r["gid"])]
    addr = lambda ip, port: (".".join(str(int(x)) for x in ip), int(port)) if int(port) else None
    off, ln = int(r["payload_off"]), int(r["payload_len"])
    return wire.Request(name, ver, int(r["req_id"]), bytes(payload[off: off + ln]), stop=bool(int(r["flags"]) & abi.F_STOP),
                        entry_replica=int(r["entry_node"]), entry_time=int(m["entry_time"]),
                        client=addr(m["client_ip"], m["client_port"]), listen=addr(m["listen_ip"], m["listen_port"]),
                        should_return=bool(int(m["flags"]) & abi.RM_RETURN_VALUE), forward_count=int(m["forward_count"]),
                        broadcasted=bool(int(m["flags"]) & abi.RM_BROADCASTED), batched=batched)


def expected_accepts(world: World, named, acc, heads, reqs, meta, payload, count=None):
    """(rstatus[count], [(gid, node, bytes)]) of the accept encoder: gpx_wire_encode_accept per sent ACCEPT, stably by
    gid, indexed once per member node that no lane serves"""
    count = len(acc) if count is None else count
    rst = np.zeros(count, np.uint8)
    sent = []
    for i in range(count):
        a = acc[i]
        gid = int(a["gid"])
        if int(a["flags"]) & abi.F_VOID or gid not in world.groups:
            rst[i] = abi.WE_VOID
        elif all(world.lane_of(m) is not None for m in world.groups[gid][2]):
            rst[i] = abi.WE_LOCAL
        elif gid not in named:
            rst[i] = abi.WE_NO_NAME
        else:
            h, nreq = int(heads[i]), int(a["nreq"])
            if nreq == 0 or h >= len(reqs) or h + nreq > len(reqs) or int(reqs[h]["gid"]) != gid:
                rst[i] = abi.WE_BAD_HEAD
            else:
                sent.append(i)
    sent.sort(key=lambda i: int(acc[i]["gid"]))
    out = []
    for i in sent:
        a = acc[i]
        gid, h, nreq = int(a["gid"]), int(heads[i]), int(a["nreq"])
        subs = tuple(to_request(world, reqs, meta, payload, q) for q in range(h + 1, h + nreq))
        b = wire.encode_accept(to_request(world, reqs, meta, payload, h, subs), int(a["slot"]), int(a["bnum"]),
                               int(a["bcoord"]), False, int(a["median_cp"]), int(a["sender"]))
        out.extend((gid, m, b) for m in world.groups[gid][2] if world.lane_of(m) is None)
    return rst, out


def random_accepts(rng, world: World, n_groups, entry_in_lanes=False):
    """(accepts, heads, reqs, meta, payload): the requests of n_groups groups grouped by gid, cut into slots of 1-5
    requests with one ACCEPT each (slots and ballots at the int32 wrap), the ACCEPTs shuffled in whole-group blocks as
    k_propose's block reservations order them, a VOID filler now and then.  entry_in_lanes: every request enters at a
    lane (its flags name the lane serving entry_node), as requests gpx_propose takes"""
    gids = sorted(int(g) for g in rng.choice(list(world.groups), size=n_groups, replace=False))
    reqs, meta, vals = [], [], []
    blocks = []
    pay_off = 0
    for gid in gids:
        name, ver, members = world.groups[gid]
        m = int(rng.integers(1, 12))
        start = len(reqs)
        for j in range(m):
            src = random_request(rng, name, ver)
            entry = int(rng.choice(world.lanes)) if entry_in_lanes else int(rng.choice(world.lanes + [7]))
            lane = world.lane_of(entry)
            rec = np.zeros(1, abi.request_dtype)[0]
            rec["gid"], rec["req_id"] = gid, src.request_id
            rec["flags"] = (abi.F_STOP if src.stop else 0) | ((0xF if lane is None else lane) << 8)
            rec["payload_off"], rec["payload_len"], rec["entry_node"], rec["client"] = pay_off, len(src.value), entry, j
            reqs.append(rec)
            meta.append(wire.req_meta(src))
            vals.append(src.value)
            pay_off += (len(src.value) + 15) & ~15
        slot = wrap32(int(rng.choice(list(SLOT_BASES.values()) + [0, 7])))
        bnum, bcoord = wrap32(BALLOT_BASE + int(rng.integers(0, 4))), int(rng.choice(members))
        block, q = [], start
        while q < start + m:
            nreq = min(int(rng.integers(1, 6)), start + m - q)
            stop = any(int(reqs[x]["flags"]) & abi.F_STOP for x in range(q, q + nreq))
            a = np.zeros(1, abi.accept_dtype)[0]
            a["gid"], a["slot"], a["bnum"], a["bcoord"], a["median_cp"] = gid, slot, bnum, bcoord, i32(rng)
            a["flags"] = abi.F_ACCEPT | (abi.F_STOP if stop else 0)
            a["dst_mask"], a["req_id"], a["nreq"], a["sender"] = world.lane_mask(gid), reqs[q]["req_id"], nreq, bcoord
            a["payload_len"] = sum(len(vals[x]) for x in range(q, q + nreq)) + (16 * nreq if nreq > 1 else 0)
            block.append((a, q))
            slot = wrap32(slot + 1)
            q += nreq
        if rng.integers(0, 4) == 0:
            v = np.zeros(1, abi.accept_dtype)[0]
            v["gid"], v["flags"] = gid, abi.F_VOID
            block.append((v, 0xFFFFFFFF))
        blocks.append(block)
    order = rng.permutation(len(blocks))
    flat = [x for k in order for x in blocks[k]]
    payload = np.zeros(max(pay_off, 16), np.uint8)
    for r, v in zip(reqs, vals):
        payload[int(r["payload_off"]): int(r["payload_off"]) + len(v)] = np.frombuffer(v, np.uint8)
    return (np.array([a for a, _ in flat], abi.accept_dtype), np.array([h for _, h in flat], np.uint32),
            np.array(reqs, abi.request_dtype), np.array(meta, abi.req_meta_dtype), payload)


def propose_blob(reqs, payload, a, head):
    """the blob gpx_propose builds for an ACCEPT whose requests are [head, head + nreq)"""
    nreq = int(a["nreq"])
    vals = [bytes(payload[int(reqs[q]["payload_off"]): int(reqs[q]["payload_off"]) + int(reqs[q]["payload_len"])])
            for q in range(head, head + nreq)]
    if nreq == 1:
        return vals[0]
    ents = np.zeros(nreq, abi.batch_ent_dtype)
    for j, q in enumerate(range(head, head + nreq)):
        ents[j] = (reqs[q]["req_id"], reqs[q]["payload_len"], reqs[q]["flags"])
    return ents.tobytes() + b"".join(vals)
