"""Cases and expectations shared by tests/test_wire_dev.py (the kernel source on the host, tests/emu/wire_emu.cpp) and
tests/test_wire_dev_gpu.py (the same kernels through the C ABI): phase-2 packets made by the host codec (gpx_wire.cpp),
what decoding them must give -- derived from the host decoders gpx_wire_decode_* and the member sets -- and a short
restatement of PaxosPacketBatcher's coalescing that feeds the host encoders to give the bytes the device encoders must
write."""
from __future__ import annotations

import struct

import numpy as np

from gigapaxos_b200 import abi, wire

LANES = (100, 101, 102)


class World:
    """groups: gid -> (name, version, sorted members); the engine's lanes serve LANES"""

    def __init__(self, groups: dict, lanes=LANES):
        self.groups = groups
        self.lanes = list(lanes)
        self.by_name = {(g[0]): gid for gid, g in groups.items()}

    def lane_mask(self, gid):
        return sum(1 << l for l, node in enumerate(self.lanes) if node in self.groups[gid][2])

    def lane_of(self, node):
        return self.lanes.index(node) if node in self.lanes else None


def random_world(rng, n_groups, lanes=LANES):
    groups = {}
    names = set()
    pool = [98, 99, 100, 101, 102, 103, 104]
    for gid in range(n_groups):
        while True:
            ln = int(rng.integers(1, 128))
            name = "".join(chr(int(c)) for c in rng.integers(33, 127, size=ln))
            if name not in names:
                break
        names.add(name)
        R = int(rng.integers(1, 6))
        members = sorted(int(x) for x in rng.choice(pool, size=R, replace=False))
        groups[gid] = (name, int(rng.integers(0, 4)), members)
    return World(groups, lanes)


def i32(rng):
    return int(rng.integers(-(1 << 31), 1 << 31))


def random_request(rng, name, version, batched=0):
    val = bytes(rng.integers(0, 256, size=int(rng.integers(0, 40))).astype(np.uint8))
    subs = tuple(random_request(rng, name, version) for _ in range(batched))
    return wire.Request(name, version, int(rng.integers(-(1 << 62), 1 << 62)), val, stop=bool(rng.integers(0, 4) == 0),
                        entry_replica=int(rng.choice([100, 101, 102, 7])), entry_time=int(rng.integers(0, 1 << 40)),
                        client=("10.0.0.1", 2000) if rng.integers(0, 2) else None, forward_count=int(rng.integers(0, 3)),
                        digest=b"d" * int(rng.integers(0, 3)), response=b"r" * int(rng.integers(0, 3)), batched=subs)


def random_packets(rng, world: World, n):
    """(packets, sources): ACCEPTs (some batched), BATCHED_ACCEPT_REPLYs and BATCHED_COMMITs with wrapping slots and
    ballots, plus a few unknown names and stale versions"""
    pkts, srcs = [], []
    gids = list(world.groups)
    for _ in range(n):
        gid = int(rng.choice(gids))
        name, ver, members = world.groups[gid]
        u = int(rng.integers(0, 20))
        if u == 0:
            name = name[:-1] + ("?" if name[-1] != "?" else "!")  # unknown (the names are random: no collision)
        elif u == 1:
            ver = ver + 1  # version mismatch
        kind = int(rng.integers(0, 3))
        base = int(rng.choice([0, (1 << 31) - 3, -5]))
        if kind == 0:
            req = random_request(rng, name, ver, batched=int(rng.integers(0, 4)) if rng.integers(0, 2) else 0)
            sender = int(rng.choice(members))
            pkts.append(wire.encode_accept(req, wrap32(base + int(rng.integers(0, 8))), i32(rng), sender, bool(rng.integers(0, 2)),
                                           i32(rng), sender))
            srcs.append(("accept", req))
        elif kind == 1:
            k = int(rng.integers(0, 9))
            slots = [wrap32(base + int(s)) for s in rng.integers(0, 12, size=k)]
            rids = [int(x) for x in rng.integers(-(1 << 62), 1 << 62, size=k)]
            acc = int(rng.choice(members + [77]))
            coord = int(rng.choice(members))
            first = slots[0] if slots else 0
            pkts.append(wire.encode_batched_accept_reply(name, ver, acc, i32(rng), coord, first, i32(rng),
                                                         rids[0] if rids else 0, slots, rids))
            srcs.append(("reply", None))
        else:
            k = int(rng.integers(0, 9))
            slots = sorted(set(wrap32(base + int(s)) for s in rng.integers(0, 12, size=k)))
            pkts.append(wire.encode_batched_commit(name, ver, i32(rng), int(rng.choice(members)), i32(rng), slots,
                                                   members))
            srcs.append(("commit", None))
    return pkts, srcs


def malformed_packets(world: World):
    """packets the decoder must classify without records"""
    gid0 = min(world.groups)
    name, ver, members = world.groups[gid0]
    good = wire.encode_batched_commit(name, ver, 1, members[0], 0, [1, 2], members)
    acc = wire.encode_accept(wire.Request(name, ver, 5, b"xy", entry_replica=members[0]), 1, 0, members[0], False, 0,
                             members[0])
    out = [
        (good[:-1], abi.WS_MALFORMED),                                   # truncated
        (good + b"\0", abi.WS_MALFORMED),                                # trailing bytes
        (b"\0\0\0\x5b" + good[4:], abi.WS_MALFORMED),                    # magic 91
        (good[:12] + b"\x80" + good[13:], abi.WS_MALFORMED),             # idLen 128
        (b"", abi.WS_MALFORMED),
        (acc[:-4], abi.WS_MALFORMED),
        (b'{"type":3}', abi.WS_UNHANDLED),                               # JSON
        (struct.pack(">iiiB", 90, 36, ver, 1) + b"x", abi.WS_UNHANDLED),  # BATCHED_ACCEPT
        (struct.pack(">iiiB", 90, 8, ver, 1) + b"x" + bytes(29), abi.WS_UNHANDLED),  # singleton ACCEPT_REPLY
        (wire.encode_batched_commit(name + "-", ver, 1, members[0], 0, [1], members), abi.WS_UNKNOWN_NAME),
        (wire.encode_batched_commit(name, ver + 7, 1, members[0], 0, [1], members), abi.WS_VERSION),
    ]
    return out


def header_of(b: bytes):
    if len(b) < 13:
        return None
    magic, ptype, ver, idl = struct.unpack(">iiiB", b[:13])
    if magic != 90 or idl > 127 or len(b) < 13 + idl:
        return None
    return ptype, ver, b[13: 13 + idl].decode("iso-8859-1")


def expected_decode(world: World, pkts, srcs=None):
    """(status, accepts, blob, replies, decisions) the decoder must produce, from the host codec's decoders"""
    status = []
    accs, reps, decs = [], [], []  # (gid, packet index, record / blob)
    for k, b in enumerate(pkts):
        if b[:1] == b"{":
            status.append(abi.WS_UNHANDLED)
            continue
        h = header_of(b)
        if h is None:
            status.append(abi.WS_MALFORMED)
            continue
        ptype, ver, name = h
        if ptype not in (wire.PT_ACCEPT, wire.PT_BATCHED_ACCEPT_REPLY, wire.PT_BATCHED_COMMIT):
            status.append(abi.WS_UNHANDLED)
            continue
        try:
            if ptype == wire.PT_ACCEPT:
                d = wire.decode_accept(b)
            elif ptype == wire.PT_BATCHED_ACCEPT_REPLY:
                d = wire.decode_batched_accept_reply(b)
            else:
                d = wire.decode_batched_commit(b)
        except ValueError:
            status.append(abi.WS_MALFORMED)
            continue
        gid = world.by_name.get(name)
        if gid is None:
            status.append(abi.WS_UNKNOWN_NAME)
            continue
        if world.groups[gid][1] != ver:
            status.append(abi.WS_VERSION)
            continue
        members = world.groups[gid][2]
        mask = world.lane_mask(gid)
        if ptype == wire.PT_BATCHED_ACCEPT_REPLY:
            if d["acceptor"] not in members or d["bcoord"] not in members:
                status.append(abi.WS_MALFORMED)
                continue
            if world.lane_of(d["bcoord"]) is None:
                status.append(abi.WS_NOT_LOCAL)
                continue
        elif mask == 0:
            status.append(abi.WS_NOT_LOCAL)
            continue
        status.append(abi.WS_OK)
        if ptype == wire.PT_ACCEPT:
            req = srcs[k][1]
            reqs = [req] + list(req.batched)
            assert d["request_id"] == req.request_id and d["n_batched"] == len(req.batched)
            assert d["value"] == req.value and bool(d["stop"]) == req.stop
            if len(reqs) == 1:
                body = d["value"]
            else:
                ents = np.zeros(len(reqs), abi.batch_ent_dtype)
                for j, r in enumerate(reqs):
                    lane = world.lane_of(r.entry_replica)
                    ents[j] = (r.request_id, len(r.value), (abi.F_STOP if r.stop else 0) | ((0xF if lane is None else lane) << 8))
                body = ents.tobytes() + b"".join(r.value for r in reqs)
            a = np.zeros(1, abi.accept_dtype)[0]
            a["gid"], a["slot"], a["bnum"], a["bcoord"], a["median_cp"] = gid, d["slot"], d["bnum"], d["bcoord"], d["median_cp"]
            a["flags"] = abi.F_ACCEPT | (abi.F_STOP if any(r.stop for r in reqs) else 0)
            a["dst_mask"], a["req_id"] = mask, d["request_id"]
            a["payload_off"], a["payload_len"], a["nreq"], a["sender"] = 0, len(body), len(reqs), d["sender"]
            accs.append((gid, k, a, body))
        elif ptype == wire.PT_BATCHED_ACCEPT_REPLY:
            who = abi.who(members.index(d["acceptor"]), members.index(d["bcoord"]), 0)
            for s, q in zip(d["slots"], d["req_ids"]):
                reps.append((gid, k, (gid, s, d["bnum"], d["bcoord"], d["max_cp"], who, q)))
        else:
            for s in d["slots"]:
                decs.append((gid, k, (gid, s, d["bnum"], d["bcoord"], d["median_cp"], abi.F_DECISION, mask, 0)))
    # grouped by gid, packet order within a gid (the lists are in packet order already: a stable sort by gid)
    accs.sort(key=lambda t: t[0])
    reps.sort(key=lambda t: t[0])
    decs.sort(key=lambda t: t[0])
    return status, accs, np.array([t[2] for t in reps], dtype=abi.reply_dtype), \
        np.array([t[2] for t in decs], dtype=abi.decision_dtype)


def check_decode(world, pkts, srcs, got):
    """got = (status, accepts, blob, replies, decisions) of a device (or emulated) decode"""
    status, acc, blob, rep, dec = got
    est, eacc, erep, edec = expected_decode(world, pkts, srcs)
    assert list(status) == est
    assert len(acc) == len(eacc)
    for a, (gid, k, ea, body) in zip(acc, eacc):
        assert int(a["payload_off"]) % 16 == 0
        got_body = bytes(blob[int(a["payload_off"]): int(a["payload_off"]) + int(a["payload_len"])])
        assert got_body == body
        for f in abi.accept_dtype.names:
            if f != "payload_off":
                assert a[f] == ea[f], f
    assert np.array_equal(rep, erep)
    assert np.array_equal(dec, edec)


# ---- PaxosPacketBatcher's coalescing, restated, over the host encoders -------------------------------------------------
def expected_encode_replies(world: World, replies: np.ndarray, n_lanes: int):
    """(rstatus, [(gid, node, bytes)]) for replies in gpx_handle_accepts' layout (i * n_lanes + lane): one
    BatchedAcceptReply per (lane, gid, ballot) run of positive replies to a remote coordinator, header from the first"""
    rstatus = np.zeros(len(replies), np.uint8)
    runs = {}  # (lane, gid) -> list of runs, each a list of record indices
    for i, r in enumerate(replies):
        fl = abi.who_flags(int(r["who"]))
        gid = int(r["gid"])
        members = world.groups[gid][2] if gid in world.groups else None
        if fl & abi.F_VOID or members is None:
            rstatus[i] = abi.WE_VOID
            continue
        if fl & abi.F_NACK:
            rstatus[i] = abi.WE_NACK
            continue
        if world.lane_of(members[abi.who_dst(int(r["who"]))]) is not None:
            rstatus[i] = abi.WE_LOCAL
            continue
        key = (i % n_lanes, gid)
        lst = runs.setdefault(key, [])
        if lst and (int(replies[lst[-1][-1]]["bnum"]), int(replies[lst[-1][-1]]["bcoord"])) == (int(r["bnum"]), int(r["bcoord"])):
            lst[-1].append(i)
        else:
            lst.append([i])
    out = []
    for key in sorted(runs, key=lambda t: (t[0], t[1])):
        for run in runs[key]:
            h = replies[run[0]]
            gid = int(h["gid"])
            name, ver, members = world.groups[gid]
            m = {}
            for i in run:  # TreeMap: last put wins
                m[int(replies[i]["slot"])] = int(replies[i]["req_id"])
            slots = sorted(m)
            b = wire.encode_batched_accept_reply(name, ver, members[abi.who_acc(int(h["who"]))], int(h["bnum"]),
                                                 int(h["bcoord"]), int(h["slot"]), int(h["max_cp"]), int(h["req_id"]),
                                                 slots, [m[s] for s in slots])
            out.append((gid, members[abi.who_dst(int(h["who"]))], b))
    return rstatus, out


def wrap32(x):
    return ((x + (1 << 31)) % (1 << 32)) - (1 << 31)


def wrap_max(a, b):
    d = (b - a) & 0xFFFFFFFF
    return b if 0 < d < (1 << 31) else a


def expected_encode_decisions(world: World, decisions: np.ndarray):
    """(rstatus, [(gid, node, bytes)]): decisions stably sorted by gid, one BatchedCommit per (gid, ballot) run with
    the wrap-aware maximum median, indexed once per member node no lane serves"""
    rstatus = np.zeros(len(decisions), np.uint8)
    keep = []
    for i, d in enumerate(decisions):
        gid = int(d["gid"])
        if int(d["flags"]) & abi.F_VOID or gid not in world.groups:
            rstatus[i] = abi.WE_VOID
        elif all(world.lane_of(m) is not None for m in world.groups[gid][2]):
            rstatus[i] = abi.WE_LOCAL
        else:
            keep.append(i)
    keep.sort(key=lambda i: int(decisions[i]["gid"]))
    out = []
    p = 0
    while p < len(keep):
        d = decisions[keep[p]]
        q = p + 1
        while q < len(keep) and int(decisions[keep[q]]["gid"]) == int(d["gid"]) and \
                (int(decisions[keep[q]]["bnum"]), int(decisions[keep[q]]["bcoord"])) == (int(d["bnum"]), int(d["bcoord"])):
            q += 1
        run = decisions[keep[p:q]]
        med = int(run[0]["median_cp"])
        for x in run[1:]:
            med = wrap_max(med, int(x["median_cp"]))
        gid = int(d["gid"])
        name, ver, members = world.groups[gid]
        b = wire.encode_batched_commit(name, ver, int(d["bnum"]), int(d["bcoord"]), med, [int(s) for s in run["slot"]],
                                       members)
        for m in members:
            if world.lane_of(m) is None:
                out.append((gid, m, b))
        p = q
    return rstatus, out


def random_replies(rng, world: World, n_accepts: int, n_lanes: int):
    """gpx_handle_accepts-shaped replies: grouped by gid, record i * n_lanes + lane"""
    gids = sorted(int(g) for g in rng.choice(list(world.groups), size=n_accepts))
    r = np.zeros(n_accepts * n_lanes, abi.reply_dtype)
    for i, gid in enumerate(gids):
        members = world.groups[gid][2]
        bn = int(rng.choice([3, 4, (1 << 31) - 1]))
        coord_idx = int(rng.integers(0, len(members)))
        for l in range(n_lanes):
            x = r[i * n_lanes + l]
            node = world.lanes[l]
            void = node not in members or rng.integers(0, 8) == 0
            fl = abi.F_VOID if void else (abi.F_NACK if rng.integers(0, 6) == 0 else 0) | (abi.F_LOGGED if rng.integers(0, 2) else 0)
            acc = members.index(node) if node in members else 0
            slot = wrap32(int(rng.choice([0, (1 << 31) - 2])) + int(rng.integers(-3, 6)))
            r[i * n_lanes + l] = (gid, slot, bn, members[coord_idx], i32(rng), abi.who(acc, coord_idx, fl),
                                  int(rng.integers(-(1 << 62), 1 << 62)))
    return r


def random_decisions(rng, world: World, n: int):
    d = np.zeros(n, abi.decision_dtype)
    gids = rng.choice(list(world.groups), size=n)
    for i, gid in enumerate(gids):
        members = world.groups[int(gid)][2]
        d[i] = (int(gid), int(rng.integers(-4, 8)), int(rng.choice([1, 2])), members[0], i32(rng),
                abi.F_DECISION | (abi.F_VOID if rng.integers(0, 10) == 0 else 0), world.lane_mask(int(gid)),
                int(rng.integers(0, 1 << 40)))
    return d
