"""The Python model of gpx_wire_encode_json_sweep_device (include/gpx.h), shared by tests/test_wire_json_sweep.py (the
kernel source on the host, tests/emu/wire_json_sweep_emu.cpp) and tests/test_wire_json_sweep_gpu.py (the C ABI on the
device).  It is built from the two models it joins: the forwarding rules of wire_fwd_cases (route, batch_end,
as_request), the reply and commit members of wire_json_out_cases, and packets_json.request_json for a forward member."""
from __future__ import annotations

import numpy as np

from gigapaxos_b200 import abi, packets_json as pj, wire
from wire_dev_cases import World, wrap_max
from wire_fwd_cases import Rows, as_request, batch_end, route
from wire_json_out_cases import (MAX_MEMBER, WRAP_BYTES, WRAP_OVERHEAD, _runs, commit_lane, decision_status,
                                 reply_status)


def forward_cuts(world: World, named, rows: Rows, reqs, meta, status, down=()):
    """(rstatus[n], [(k, b, gid, destination, sending lane)] for every GPX_WE_SENT cut, in request order): the walk of
    wire_fwd_cases.expected_forwards, keeping the cuts"""
    n = len(reqs)
    rst = np.full(n, abi.WE_VOID, np.uint8)
    cuts = []
    i = 0
    while i < n:
        gid = int(reqs[i]["gid"])
        e = i + 1
        while e < n and int(reqs[e]["gid"]) == gid:
            e += 1
        lane = (int(reqs[i]["flags"]) >> 8) & 0xF
        code, bc = route(world, rows, gid, lane)
        routed = code == abi.RS_FORWARD
        run_st, dst = abi.WE_SENT, bc
        if routed:
            members = world.groups[gid][2]
            if bc not in members:
                run_st = abi.WE_ELECT
            else:
                di = members.index(bc)
                if bc in down:
                    di = (di + 1) % len(members)
                dst = members[di]
                if dst in world.lanes:
                    run_st = abi.WE_ELECT
        fwd = lambda q: int(status[q]) == abi.RS_FORWARD and not int(meta[q]["flags"]) & abi.RM_BROADCASTED
        k = i
        while k < e:
            if not routed or not fwd(k):
                k += 1
                continue
            b = min(batch_end(rows, reqs, k, gid), e)
            c = k + 1
            while c < b and fwd(c):
                c += 1
            b = c
            st = run_st
            if st == abi.WE_SENT and forward_count(meta, k) > 3:
                st = abi.WE_ELECT
            if st == abi.WE_SENT and gid not in named:
                st = abi.WE_NO_NAME
            rst[k:b] = st
            if st == abi.WE_SENT:
                cuts.append((k, b, gid, dst, lane))
            k = b
        i = e
    return rst, cuts


def forward_count(meta, k):
    """forwardCount + 1 as a Java int"""
    return ((int(meta[k]["forward_count"]) + 1 + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def forward_packet(world: World, reqs, meta, payload, k, b) -> bytes:
    """gpx_wire_encode_request of the cut [k, b): the outer request with forwardCount + 1, the others its batched"""
    outer = as_request(world, reqs[k], meta[k], payload, forward_count=forward_count(meta, k))
    outer.batched = tuple(as_request(world, reqs[q], meta[q], payload) for q in range(k + 1, b))
    return wire.encode_request(outer)


def forward_member(world: World, reqs, meta, payload, k) -> bytes:
    return pj.request_json(as_request(world, reqs[k], meta[k], payload, forward_count=forward_count(meta, k)))


def expected_sweep(world: World, named, replies, decisions, fwd=None, n_dec=None, wrap_bytes=WRAP_BYTES):
    """fwd = (rows, reqs, meta, status, payload, down) or None -> (rstatus_replies, rstatus_decisions[:n_dec],
    rstatus_reqs, out bytes, [(off, len, gid, node)], [(k, b) of each lone packet]) the call must produce"""
    L = len(world.lanes)
    replies = np.zeros(0, abi.reply_dtype) if replies is None else replies
    decisions = np.zeros(0, abi.decision_dtype) if decisions is None else decisions
    n_dec = len(decisions) if n_dec is None else n_dec
    rst_r = np.array([reply_status(world, named, r) for r in replies], np.uint8)
    rst_d = np.array([decision_status(world, named, d) for d in decisions[:n_dec]], np.uint8)
    packets = []  # (bytes, gid, [nodes])
    for i, r in enumerate(replies):
        if rst_r[i] == abi.WE_NACK:
            gid = int(r["gid"])
            name, ver, members = world.groups[gid]
            who = int(r["who"])
            packets.append((pj.accept_reply_json(name, ver, members[abi.who_acc(who)], int(r["bnum"]), int(r["bcoord"]),
                                                 int(r["slot"]), int(r["max_cp"]), int(r["req_id"])),
                            gid, [members[abi.who_dst(who)]]))
    # forwards: a cut of one request that fits is a member of its entry lane's sweep, every other cut goes alone
    seq = {l: [] for l in range(L)}
    rst_q, lone, fwd_members = np.zeros(0, np.uint8), [], []
    if fwd is not None:
        rows, reqs, meta, status, payload, down = fwd
        rst_q, cuts = forward_cuts(world, named, rows, reqs, meta, status, down)
        for k, b, gid, dst, lane in cuts:
            obj = forward_member(world, reqs, meta, payload, k) if b - k == 1 else None
            if obj is not None and len(obj) <= MAX_MEMBER:
                fwd_members.append((lane, ("q", frozenset([dst]), obj)))
            else:
                packets.append((forward_packet(world, reqs, meta, payload, k, b), gid, [dst]))
                lone.append((k, b))
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
        seq[lane].append(("d", frozenset(x for x in members if world.lane_of(x) is None), obj))
    for lane, m in fwd_members:
        seq[lane].append(m)
    T = wrap_bytes - WRAP_OVERHEAD - MAX_MEMBER
    for lane in range(L):
        ordered = [x for kind in "rdq" for x in seq[lane] if x[0] == kind]  # dequeueImpl's order
        groups = {}
        for _, rs, obj in ordered:  # first-seen order (LinkedHashMap)
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
    return rst_r, rst_d, rst_q, out, refs, lone


def coordinator_world(lanes=(100, 101, 102)):
    """groups whose acceptors at lane 0 (node 100) reply to coordinator 103 and forward to it: group 0 {100, 103},
    group 1 {100, 101, 103}, group 2 {100, 104} (its coordinator 104)"""
    return World({0: ("fw-a", 0, [100, 103]), 1: ("fw-b", 2, [100, 101, 103]), 2: ("fw-c", 0, [100, 104])}, list(lanes))
