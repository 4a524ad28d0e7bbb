"""Cases and expectations shared by tests/test_wire_forward.py (the forwarding kernels on the host,
tests/emu/wire_fwd_emu.cpp) and tests/test_wire_forward_gpu.py (the same kernels through the C ABI):

* JSON forms of RequestPackets -- every QV byte written raw, escaped or as \\u00XX, '/' sometimes as \\/ -- inside
  BATCHED_PAXOS_PACKET wrappers beside reply and commit members, and a malformed / host-only corpus with a Python model
  of the schema;
* a restatement of the forwarding rules (propose_run's routing, RequestBatcher's cut, getNextCoordinator, the
  ping-pong and local-coordinator checks) that feeds gpx_wire_encode_request to give the bytes the encoder must write."""
from __future__ import annotations

import json
import re

import numpy as np

from gigapaxos_b200 import abi, packets_json as pj, wire
from wire_dev_cases import World

I32 = (-(1 << 31), (1 << 31) - 1)
I64 = (-(1 << 63), (1 << 63) - 1)
ESC = {8: b"\\b", 9: b"\\t", 10: b"\\n", 12: b"\\f", 13: b"\\r"}


# ---- JSON forms --------------------------------------------------------------------------------------------------------
def json_string(b: bytes, rng) -> bytes:
    """a JSON string of the ISO-8859-1 characters b, each written one of the ways a JSON writer may write it"""
    out = bytearray(b'"')
    for c in b:
        r = int(rng.integers(0, 3))
        if c == 0x22:
            out += b'\\"' if r else b"\\u0022"
        elif c == 0x5C:
            out += b"\\\\" if r else b"\\u005C"
        elif c == 0x2F:
            out += b"\\/" if r == 1 else b"/"
        elif c < 0x20:
            out += ESC.get(c, b"\\u%04x" % c) if r else b"\\u%04X" % c
        elif r or c == 0x7F:
            out += bytes([c])  # raw, 0x80-0xff included: an ISO-8859-1 byte
        else:
            out += b"\\u%04x" % c
    return bytes(out + b'"')


def request_member(r: wire.Request, rng) -> bytes:
    """packets_json.request_json's object for r, its QV values written by json_string"""
    d = pj._request_smart(r, pj.PT_REQUEST)
    vals = []

    def mark(o, req):
        o["QV"] = "\0QV%d" % len(vals)
        vals.append(req.value)
        for so, sr in zip(o.get("BATCH", []), req.batched):
            mark(so, sr)
    mark(d, r)
    b = json.dumps(d, separators=(",", ":")).encode("ascii")
    for k, v in enumerate(vals):
        b = b.replace(b'"\\u0000QV%d"' % k, json_string(v, rng), 1)
    return b


def wrapper(members) -> bytes:
    return b'{"type":90,"PT":37,"V":-1,"PP":[' + b",".join(members) + b"]}"


def filler_member(world: World, rng) -> bytes:
    gid = int(rng.choice(list(world.groups)))
    name, ver, members = world.groups[gid]
    if rng.integers(0, 2):
        return pj.batched_accept_reply_json(name, ver, members[0], 3, members[-1], 5, 0, 9, [5, 6], [9, 10])
    return pj.batched_commit_json(name, ver, 3, members[-1], 0, [5, 6], members)


def json_wrappers(world: World, pkts, rng):
    """pkts [(bytes, node, Request)] -> (wrappers [(bytes, node)], order): the requests as JSON members of wrappers
    received at their node, 1-5 to a wrapper, among reply and commit members; order[j] = (packet index, member index)
    of the j-th REQUEST member in member order"""
    by_node = {}
    for k, (_, node, req) in enumerate(pkts):
        by_node.setdefault(node, []).append(k)
    wraps, order, m = [], [], 0
    for node, ks in by_node.items():
        i = 0
        while i < len(ks):
            take = ks[i: i + int(rng.integers(1, 6))]
            i += len(take)
            members = []
            for k in take:
                if rng.integers(0, 3) == 0:
                    members.append(filler_member(world, rng))
                order.append((k, m + len(members)))
                members.append(request_member(pkts[k][2], rng))
            m += len(members)
            wraps.append((wrapper(members), node))
    return wraps, order


# ---- the schema model ----------------------------------------------------------------------------------------------
def _int(v, lim):
    return type(v) is int and lim[0] <= v <= lim[1]


def _addr_literal(s: str) -> bool:
    if any(c in s for c in "\n\r\x85") or any(ord(c) > 0xFF for c in s):
        return False
    t = s.rsplit("/", 1)[-1]
    m = re.fullmatch(r"(0|[1-9][0-9]{0,2})\.(0|[1-9][0-9]{0,2})\.(0|[1-9][0-9]{0,2})\.(0|[1-9][0-9]{0,2}):([0-9]{1,5})", t)
    return bool(m) and all(int(x) <= 255 for x in m.groups()[:4]) and 1 <= int(m.group(5)) <= 65535


def model_fields(d: dict, top: bool):
    """WS_OK / WS_MALFORMED / WS_UNHANDLED of one request object's fields (RequestPacket(JSONObject) :584-649)"""
    ok = (_int(d.get("QID"), I64) and type(d.get("QV")) is str and _int(d.get("ET"), I64)
          and _int(d.get("E"), I32))
    ok = ok and ("NFWDS" not in d or _int(d["NFWDS"], I32))
    ok = ok and all(type(d[k]) is bool for k in ("STOP", "QF", "BC") if k in d)
    ok = ok and all(type(d[k]) is str for k in ("CA", "LA") if k in d)
    host = ok and ("RV" in d or "DIG" in d or any(ord(c) > 0xFF for c in d["QV"])
                   or not all(_addr_literal(d[k]) for k in ("CA", "LA") if k in d))
    if ok and top and "BATCH" in d:
        b = d["BATCH"]
        ok = type(b) is list and all(type(x) is dict and "BATCH" not in x for x in b)
        if ok:
            subs = [model_fields(x, False) for x in b]
            ok = abi.WS_MALFORMED not in subs
            host = host or abi.WS_UNHANDLED in subs
    if not ok:
        return abi.WS_MALFORMED
    return abi.WS_UNHANDLED if host else abi.WS_OK


def malformed_corpus(world: World):
    """[(member bytes, node, expected status)]: one member per wrapper, its status from model_fields"""
    gid = min(g for g in world.groups if any(m in world.lanes for m in world.groups[g][2]))
    name, ver, members = world.groups[gid]
    node = next(m for m in members if m in world.lanes)
    good = json.loads(pj.request_json(wire.Request(name, ver, 5, b"xy", entry_replica=node,
                                                   batched=(wire.Request(name, ver, 6, b"z"),))))

    def v(**kw):
        d = dict(good)
        for k, x in kw.items():
            if x is KeyError:
                d.pop(k, None)
            else:
                d[k] = x
        return d
    sub = good["BATCH"][0]
    objs = [v(E=KeyError), v(ET=KeyError), v(QID=KeyError), v(QV=KeyError),
            v(QID="5"), v(ET=1.5), v(E=True), v(QV=7), v(NFWDS=1 << 31), v(NFWDS=-(1 << 31) - 1), v(STOP=1),
            v(QF="true"), v(CA=5), v(BATCH=3), v(BATCH=[1]), v(BATCH=[dict(sub, BATCH=[])]), v(BATCH=[dict(sub, E=None)]),
            v(CA="host.example:80"), v(CA="/[::1]:80"), v(LA="/1.2.3.4:0"), v(LA="/1.2.3.4:65536"),
            v(CA="/01.2.3.4:80"), v(CA="a\nb/1.2.3.4:80"), v(CA="/1.2.3.4"), v(QV="xĀ"),
            v(BATCH=[dict(sub, QV="€")]), v(RV=""), v(DIG="d"), v(BATCH=[dict(sub, RV="r")]),
            v(CA="some.host/10.1.2.3:80", LA="/0.0.0.0:65535"), v(NFWDS=(1 << 31) - 1), v(QID=I64[0], ET=I64[1]),
            v(E=-1), v(BATCH=[]), v(FWDR=7, DBG="x", UNKNOWN={"a": [1, {"b": None}]}), v(PT=3), good]
    raw = [json.dumps(o, separators=(",", ":")).encode("ascii") for o in objs]
    out = [(b, node, abi.WS_UNHANDLED if o["PT"] != pj.PT_REQUEST else model_fields(o, True)) for b, o in zip(raw, objs)]
    # valid JSON numbers that are not integers, an int64 out of range (a leading zero or '+' is not JSON: the wrapper
    # is malformed before any member is listed)
    q = pj.request_json(wire.Request(name, ver, 5, b"xy", entry_replica=node))
    for bad in (b'"E":1.0', b'"E":1e2', b'"E":-0.5'):
        out.append((q.replace(b'"E":%d' % node, bad), node, abi.WS_MALFORMED))
    out.append((q.replace(b'"ET":0', b'"ET":9223372036854775808'), node, abi.WS_MALFORMED))
    out.append((q.replace(b'"QID":5', b'"QID":5,"QID":-9'), node, abi.WS_OK))  # the last duplicate counts
    return out


# ---- forwarding ---------------------------------------------------------------------------------------------------------
class Rows:
    """the acceptor and coordinator rows the routing reads, [L][G] each, and RequestBatcher's settings"""

    def __init__(self, L, G, batching=1, max_batch_size=5, size_est=0, max_batch_bytes=1 << 30):
        self.acc = np.zeros((L, G, 4), np.int32)
        self.aux = np.full((L, G), abi.ST_ACTIVE_1, np.uint32)
        self.coord = np.zeros((L, G, 4), np.int32)
        self.batching, self.max_batch_size, self.size_est = batching, max_batch_size, size_est
        self.max_batch_bytes = max_batch_bytes


def route(world: World, rows: Rows, gid, entry):
    """propose_route: (code, ballot coordinator)"""
    if gid not in world.groups or entry >= len(world.lanes) or rows.aux[entry, gid] not in (1, 2):
        return abi.RS_DROPPED, 0
    A, Cr = rows.acc[entry, gid], rows.coord[entry, gid]
    bc = int(A[2])

    def exists(a, c):
        return (int(c[3]) & 1) and bcmp(int(c[0]), int(c[1]), int(a[1]), int(a[2])) >= 0
    if exists(A, Cr):
        return 0, bc
    fl = world.lane_of(bc)
    if fl is None:
        return abi.RS_FORWARD, bc
    if fl == entry or rows.aux[fl, gid] not in (1, 2):
        return (abi.RS_NOCOORD if fl == entry else abi.RS_DROPPED), bc
    return (0 if exists(rows.acc[fl, gid], rows.coord[fl, gid]) else abi.RS_NOCOORD), bc


def jsub(a, b):
    return ((a - b + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def bcmp(an, ac, bn, bc):
    return jsub(an, bn) if an != bn else jsub(ac, bc)


def batch_end(rows: Rows, reqs, k, gid):
    n = len(reqs)
    nbytes, cnt, b = int(reqs[k]["payload_len"]) + rows.size_est, 1, k + 1
    if rows.batching:
        while b < n and int(reqs[b]["gid"]) == gid:
            nbytes += int(reqs[b]["payload_len"]) + rows.size_est
            if nbytes > rows.max_batch_bytes:
                break
            cnt += 1
            if cnt > rows.max_batch_size:
                break
            b += 1
    return b


def as_request(world: World, rec, m, payload, forward_count=None) -> wire.Request:
    name, ver, _ = world.groups[int(rec["gid"])]
    addr = lambda ip, port: (".".join(str(int(x)) for x in ip), int(port)) if int(port) else None
    off, ln = int(rec["payload_off"]), int(rec["payload_len"])
    return wire.Request(name, ver, int(rec["req_id"]), bytes(payload[off: off + ln]),
                        stop=bool(int(rec["flags"]) & abi.F_STOP), entry_replica=int(rec["entry_node"]),
                        entry_time=int(m["entry_time"]), client=addr(m["client_ip"], m["client_port"]),
                        listen=addr(m["listen_ip"], m["listen_port"]),
                        should_return=bool(int(m["flags"]) & abi.RM_RETURN_VALUE),
                        forward_count=int(m["forward_count"]) if forward_count is None else forward_count,
                        broadcasted=bool(int(m["flags"]) & abi.RM_BROADCASTED))


def expected_forwards(world: World, named, rows: Rows, reqs, meta, status, payload, down=()):
    """(rstatus[n], [(gid, node, bytes)] in request order) gpx_wire_encode_forwards_device must give"""
    n = len(reqs)
    rst = np.full(n, abi.WE_VOID, np.uint8)
    out = []
    i = 0
    while i < n:
        gid = int(reqs[i]["gid"])
        e = i + 1
        while e < n and int(reqs[e]["gid"]) == gid:
            e += 1
        code, bc = route(world, rows, gid, (int(reqs[i]["flags"]) >> 8) & 0xF)
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
            fc = ((int(meta[k]["forward_count"]) + 1 + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)
            st = run_st
            if st == abi.WE_SENT and fc > 3:
                st = abi.WE_ELECT
            if st == abi.WE_SENT and gid not in named:
                st = abi.WE_NO_NAME
            rst[k:b] = st
            if st == abi.WE_SENT:
                outer = as_request(world, reqs[k], meta[k], payload, forward_count=fc)
                outer.batched = tuple(as_request(world, reqs[q], meta[q], payload) for q in range(k + 1, b))
                out.append((gid, dst, wire.encode_request(outer)))
            k = b
        i = e
    return rst, out


def forward_case(rng, world: World, n_req, L=3, **rows_kw):
    """(rows, reqs, meta, status, payload, down): grouped requests entering at random lanes; per group a ballot whose
    coordinator is a remote member, a local lane, or no member at all, and sometimes a coordinator at the entry lane; the
    statuses propose_run would give, except that some requests of locally routed runs carry -2 (a wrapped slot) and a
    few forwarded ones were given another status"""
    G = max(world.groups) + 1
    rows = Rows(L, G, **rows_kw)
    pool = [98, 99, 100, 101, 102, 103, 104, 105]
    for gid, (_, _, members) in world.groups.items():
        remote = [m for m in members if m not in world.lanes]
        for l in range(L):
            bc = int(rng.choice(remote)) if remote and rng.integers(0, 4) else int(rng.choice(members + [int(rng.choice(pool))]))
            rows.acc[l, gid] = (0, int(rng.integers(-3, 3)), bc, 0)
            if rng.integers(0, 4) == 0:  # a coordinator at this lane, its ballot at or above the acceptor's
                rows.coord[l, gid] = (rows.acc[l, gid][1] + int(rng.integers(0, 2)), rows.acc[l, gid][2], 0, 3)
            if rng.integers(0, 15) == 0:
                rows.aux[l, gid] = abi.ST_STOPPED
    gids = np.sort(rng.choice(list(world.groups), size=n_req))
    reqs = np.zeros(n_req, abi.request_dtype)
    meta = np.zeros(n_req, abi.req_meta_dtype)
    lens = rng.integers(0, 24, size=n_req)
    offs = np.concatenate([[0], np.cumsum((lens + 15) // 16 * 16)[:-1]]).astype(np.uint32)
    payload = rng.integers(0, 256, size=int(offs[-1] + 32)).astype(np.uint8)
    entry_of = {int(g): int(rng.integers(0, L)) for g in set(gids.tolist())}
    for q, g in enumerate(gids):
        reqs[q]["gid"] = g
        reqs[q]["flags"] = (entry_of[int(g)] << 8) | (abi.F_STOP if rng.integers(0, 8) == 0 else 0)
        reqs[q]["req_id"] = int(rng.integers(-(1 << 62), 1 << 62))
        reqs[q]["payload_off"], reqs[q]["payload_len"] = offs[q], lens[q]
        reqs[q]["entry_node"] = int(rng.choice([100, 101, 102, 7]))
        reqs[q]["client"] = q
        addr = [None, ("10.0.0.1", 2000), ("1.2.3.4", 65535)]
        r = wire.Request("x", 0, 0, b"", client=addr[int(rng.integers(0, 3))], listen=addr[int(rng.integers(0, 3))],
                         should_return=bool(rng.integers(0, 2)), broadcasted=rng.integers(0, 12) == 0,
                         forward_count=int(rng.choice([0, 0, 1, 2, 3, 4, -1, (1 << 31) - 1])),
                         entry_time=int(rng.integers(0, 1 << 41)))
        meta[q] = wire.req_meta(r)
    status = np.zeros(n_req, np.int32)
    for q in range(n_req):
        code, _ = route(world, rows, int(gids[q]), entry_of[int(gids[q])])
        if code == 0:
            status[q] = -2 if rng.integers(0, 3) == 0 else int(rng.integers(-100, 100))
        else:
            status[q] = code
            if code == abi.RS_FORWARD and rng.integers(0, 12) == 0:
                status[q] = abi.RS_BACKPRESSURE
    down = [int(x) for x in rng.choice(pool, size=2, replace=False)]
    return rows, reqs, meta, status, payload, down
