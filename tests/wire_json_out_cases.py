"""Cases and the Python model of gpx_wire_encode_json_device (include/gpx.h), shared by tests/test_wire_json_out.py (the
kernel source on the host, tests/emu/wire_json_out_emu.cpp) and tests/test_wire_json_out_gpu.py (the C ABI on the
device).  The model is built from packets_json's objects only: the statuses, the members (one per run, as the byte
encoders cut runs), the sweep per lane, the grouping by recipient set in first-seen order, the cut rule and the refs."""
from __future__ import annotations

import numpy as np

from gigapaxos_b200 import abi, packets_json as pj
from wire_dev_cases import World, i32, random_world, wrap32, wrap_max

WRAP_BYTES = 4 << 20
WRAP_OVERHEAD = 34
MAX_MEMBER = 65536
I64_EDGES = [-(1 << 63), (1 << 63) - 1, -1, 0]


def _lane_of(world: World, node):
    return world.lane_of(node)


def reply_status(world: World, named, r):
    fl = abi.who_flags(int(r["who"]))
    gid = int(r["gid"])
    if fl & abi.F_VOID:
        return abi.WE_VOID
    if gid not in world.groups:
        return abi.WE_VOID
    members = world.groups[gid][2]
    dst, acc = abi.who_dst(int(r["who"])), abi.who_acc(int(r["who"]))
    if dst >= len(members) or acc >= len(members):
        return abi.WE_VOID
    if _lane_of(world, members[dst]) is not None:
        return abi.WE_LOCAL
    if gid not in named:
        return abi.WE_NO_NAME
    return abi.WE_NACK if fl & abi.F_NACK else abi.WE_SENT


def decision_status(world: World, named, d):
    gid = int(d["gid"])
    if int(d["flags"]) & abi.F_VOID or gid not in world.groups:
        return abi.WE_VOID
    if all(_lane_of(world, m) is not None for m in world.groups[gid][2]):
        return abi.WE_LOCAL
    if gid not in named:
        return abi.WE_NO_NAME
    return abi.WE_SENT


def _runs(order, recs):
    """consecutive entries of `order` (a stable key order) with the same key and ballot"""
    runs = []
    for key, i in order:
        r = recs[i]
        if runs and runs[-1][0] == key and (int(recs[runs[-1][1][-1]]["bnum"]), int(recs[runs[-1][1][-1]]["bcoord"])) == \
                (int(r["bnum"]), int(r["bcoord"])):
            runs[-1][1].append(i)
        else:
            runs.append((key, [i]))
    return runs


def commit_lane(world: World, members, bcoord):
    if bcoord in members and _lane_of(world, bcoord) is not None:
        return _lane_of(world, bcoord)
    local = [l for l, node in enumerate(world.lanes) if node in members]
    return min(local) if local else 0


def expected_json(world: World, named, replies, decisions, n_dec=None, wrap_bytes=WRAP_BYTES):
    """(rstatus_replies, rstatus_decisions[:n_dec], out bytes, [(off, len, gid, node)]) the call must produce"""
    L = len(world.lanes)
    replies = np.zeros(0, abi.reply_dtype) if replies is None else replies
    decisions = np.zeros(0, abi.decision_dtype) if decisions is None else decisions
    n_dec = len(decisions) if n_dec is None else n_dec
    rst_r = np.array([reply_status(world, named, r) for r in replies], np.uint8)
    rst_d = np.array([decision_status(world, named, d) for d in decisions[:n_dec]], np.uint8)
    # bare NACKs, record order
    packets = []  # (bytes, gid, [nodes])
    for i, r in enumerate(replies):
        if rst_r[i] == abi.WE_NACK:
            gid = int(r["gid"])
            name, ver, members = world.groups[gid]
            who = int(r["who"])
            packets.append((pj.accept_reply_json(name, ver, members[abi.who_acc(who)], int(r["bnum"]), int(r["bcoord"]),
                                                 int(r["slot"]), int(r["max_cp"]), int(r["req_id"])),
                            gid, [members[abi.who_dst(who)]]))
    # members: (lane, recipients, bytes) in sweep order per lane
    seq = {l: [] for l in range(L)}
    rorder = sorted(((i % L, int(replies[i]["gid"])), i) for i in range(len(replies)) if rst_r[i] == abi.WE_SENT)
    for (lane, gid), run in _runs(rorder, replies):
        h = replies[run[0]]
        name, ver, members = world.groups[gid]
        m = {}
        for i in run:
            m[int(replies[i]["slot"])] = int(replies[i]["req_id"])
        who = int(h["who"])
        obj = pj.batched_accept_reply_json(name, ver, members[abi.who_acc(who)], int(h["bnum"]), int(h["bcoord"]),
                                           int(h["slot"]), int(h["max_cp"]), int(h["req_id"]), list(m), list(m.values()))
        seq[lane].append(("r", frozenset([members[abi.who_dst(who)]]), obj))
    dorder = sorted((int(decisions[i]["gid"]), i) for i in range(n_dec) if rst_d[i] == abi.WE_SENT)
    for gid, run in _runs(dorder, decisions):
        d = decisions[run[0]]
        name, ver, members = world.groups[gid]
        med = int(d["median_cp"])
        for i in run[1:]:
            med = wrap_max(med, int(decisions[i]["median_cp"]))
        obj = pj.batched_commit_json(name, ver, int(d["bnum"]), int(d["bcoord"]), med,
                                     [int(decisions[i]["slot"]) for i in run], members)
        lane = commit_lane(world, members, int(d["bcoord"]))
        seq[lane].append(("d", frozenset(x for x in members if _lane_of(world, x) is None), obj))
    T = wrap_bytes - WRAP_OVERHEAD - MAX_MEMBER
    for lane in range(L):
        ordered = [x for x in seq[lane] if x[0] == "r"] + [x for x in seq[lane] if x[0] == "d"]
        groups = {}
        for _, rs, obj in ordered:  # dict: first-seen order (LinkedHashMap)
            groups.setdefault(rs, []).append(obj)
        for rs, objs in groups.items():
            start, cur, prev_w = 0, [], None
            for obj in objs:
                w = start // T
                if cur and w != prev_w:
                    packets.append((pj.batched_paxos_packet_json(cur), lane, sorted(rs)))
                    cur = []
                cur.append(obj)
                prev_w = w
                start += len(obj) + 1
            packets.append((pj.batched_paxos_packet_json(cur), lane, sorted(rs)))
    out, refs, off = b"", [], 0
    for b, gid, nodes in packets:
        for node in nodes:
            refs.append((off, len(b), gid, node))
        out += b
        off += len(b)
    return rst_r, rst_d, out, refs


# ---- worlds ------------------------------------------------------------------------------------------------------------
def hard_name(rng, k, max_len=127):
    """names with quotes, backslashes, control characters, 0x7f and bytes >= 0x80 (ISO-8859-1), up to max_len bytes"""
    ln = int(rng.integers(1, max_len + 1)) if k % 5 else max_len
    pool = [0x22, 0x5C, 0x08, 0x0C, 0x0A, 0x0D, 0x09, 0x00, 0x01, 0x1F, 0x7F, 0x80, 0xE9, 0xFF, 0x2F]
    chars = [int(rng.choice(pool)) if rng.integers(0, 3) == 0 else int(rng.integers(0x20, 0x7F)) for _ in range(ln)]
    return "".join(chr(c) for c in chars) + f"#{k}"[: max(0, max_len - ln)]


def json_world(rng, n_groups, lanes, permute=True):
    """wire_dev_cases.random_world with hard names and, when permute, member lists that are permutations of others
    (the member-set table keeps them as distinct sets)"""
    base = random_world(rng, n_groups, lanes)
    groups = {}
    seen = set()
    for gid, (name, ver, members) in base.groups.items():
        while True:
            nm = hard_name(rng, gid)
            if nm not in seen and len(nm.encode("iso-8859-1")) <= 127:
                break
        seen.add(nm)
        ms = list(members)
        if permute and len(ms) > 1 and rng.integers(0, 3) == 0:
            ms = list(rng.permutation(ms))
            ms = [int(x) for x in ms]
        groups[gid] = (nm, ver, ms)
    return World(groups, lanes)


def json_replies(rng, world: World, n_accepts: int, n_lanes: int):
    """gpx_handle_accepts-shaped replies with NACKs, VOIDs, ballots and slots at the int32 wrap and int64 req_ids"""
    gids = sorted(int(g) for g in rng.choice(list(world.groups), size=n_accepts))
    r = np.zeros(n_accepts * n_lanes, abi.reply_dtype)
    for i, gid in enumerate(gids):
        members = world.groups[gid][2]
        bn = int(rng.choice([3, 4, (1 << 31) - 1, -(1 << 31)]))
        coord_idx = int(rng.integers(0, len(members)))
        for l in range(n_lanes):
            node = world.lanes[l]
            void = node not in members or rng.integers(0, 8) == 0
            fl = abi.F_VOID if void else (abi.F_NACK if rng.integers(0, 6) == 0 else 0) | (abi.F_LOGGED if rng.integers(0, 2) else 0)
            acc = members.index(node) if node in members else 0
            slot = wrap32(int(rng.choice([0, (1 << 31) - 2, -(1 << 31)])) + int(rng.integers(-3, 6)))
            q = int(rng.choice(I64_EDGES)) if rng.integers(0, 4) == 0 else int(rng.integers(-(1 << 62), 1 << 62))
            r[i * n_lanes + l] = (gid, slot, bn, members[coord_idx], i32(rng), abi.who(acc, coord_idx, fl), q)
    return r


def json_decisions(rng, world: World, n: int):
    d = np.zeros(n, abi.decision_dtype)
    gids = sorted(int(g) for g in rng.choice(list(world.groups), size=n)) if rng.integers(0, 2) else \
        [int(g) for g in rng.choice(list(world.groups), size=n)]
    for i, gid in enumerate(gids):
        members = world.groups[gid][2]
        d[i] = (gid, wrap32(int(rng.choice([0, (1 << 31) - 3])) + int(rng.integers(-4, 8))),
                int(rng.choice([1, 2, (1 << 31) - 1])), int(rng.choice(members)), i32(rng),
                abi.F_DECISION | (abi.F_VOID if rng.integers(0, 10) == 0 else 0), world.lane_mask(gid),
                int(rng.integers(0, 1 << 40)))
    return d


def coordinator_commit_world(lanes):
    """two groups on the same nodes in different orders, and a group whose only remote member is the coordinator the
    replies of the first two go to: their replies and its commits share one recipient set"""
    a, b = lanes[0], lanes[1] if len(lanes) > 1 else lanes[0]
    groups = {0: ("perm-a", 0, [a, 103, 104]), 1: ("perm-b", 0, [104, a, 103]), 2: ("coord", 0, sorted({a, b, 103}))}
    return World(groups, lanes)
