"""Cases shared by tests/test_wire_json.py (the JSON decoder's kernel source on the host, tests/emu/wire_json_emu.cpp)
and tests/test_wire_json_gpu.py (the same kernels through gpx_wire_decode_json_device): logical BatchedAcceptReplies,
BatchedCommits and singleton ACCEPT_REPLYs in both their byte and their JSON forms, JSON re-serialised with shuffled keys,
whitespace, escapes and unknown keys, wrappers with known member spans, and a small Python model of the schema that
says what the decoder must make of any packet."""
from __future__ import annotations

import json

import numpy as np

from gigapaxos_b200 import abi, packets_json as pj, wire
from wire_dev_cases import World, wrap32

WS = [b"", b" ", b"\n", b"\t", b"\r\n  "]


def _jstr(s: str, rng=None) -> bytes:
    """a JSON string of s, ISO-8859-1 bytes; with rng some characters escaped (\\/, \\u00XX) or left raw above 0x7f"""
    out = bytearray(b'"')
    for ch in s:
        o = ord(ch)
        if ch in '"\\':
            out += b"\\" + ch.encode()
        elif o < 0x20 or o > 0xFF:
            out += b"\\u%04x" % o
        elif rng is not None and ch == "/" and rng.integers(0, 2):
            out += b"\\/"
        elif rng is not None and rng.integers(0, 6) == 0:
            out += (b"\\u%04X" if rng.integers(0, 2) else b"\\u%04x") % o
        else:
            out += bytes([o])
    return bytes(out + b'"')


def _junk(rng, depth=0):
    u = int(rng.integers(0, 6 if depth < 3 else 4))
    if u == 0:
        return int(rng.integers(-10**12, 10**12))
    if u == 1:
        return float(rng.integers(0, 100)) / 8 + 1e-3
    if u == 2:
        return "x/é\"\\" + str(int(rng.integers(0, 9)))
    if u == 3:
        return [None, True, False][int(rng.integers(0, 3))]
    if u == 4:
        return [_junk(rng, depth + 1) for _ in range(int(rng.integers(0, 4)))]
    return {"k%d" % i: _junk(rng, depth + 1) for i in range(int(rng.integers(0, 3)))}


def dumps_var(d: dict, rng) -> bytes:
    """d as JSON with shuffled keys, random whitespace, escaped / raw Latin-1 strings, unknown keys with nested values,
    and duplicated keys whose earlier value is junk"""
    ws = lambda: WS[int(rng.integers(0, len(WS)))]
    items = list(d.items())
    for i in range(int(rng.integers(0, 3))):
        items.append(("zz%d" % i, _junk(rng)))
    for k in list(d)[: int(rng.integers(0, 3))]:
        items.insert(0, (k, _junk(rng)))  # an earlier duplicate: the last value counts
    order = list(range(len(items)))
    rng.shuffle(order)
    # keep each duplicate's real value after its junk one
    seen, parts = {}, []
    for i, (k, v) in enumerate(items):
        seen.setdefault(k, []).append(i)
    ordered = [items[seen[items[i][0]].pop(0)] for i in order]
    for k, v in ordered:
        if isinstance(v, str):
            val = _jstr(v, rng)
        else:
            val = json.dumps(v, ensure_ascii=False).encode("iso-8859-1", errors="backslashreplace")
        parts.append(ws() + _jstr(k) + ws() + b":" + ws() + val + ws())
    return b"{" + b",".join(parts) + b"}" if parts else b"{" + ws() + b"}"


def wrap(members, rng=None):
    """a BATCHED_PAXOS_PACKET of member JSON bytes -> (packet, [(offset, length)] of each member in it)"""
    ws = (lambda: WS[int(rng.integers(0, len(WS)))]) if rng is not None else (lambda: b"")
    head = b"{" + ws() + b'"type"' + ws() + b":90," + ws() + b'"PT":37,"V"' + ws() + b":" + ws() + b"-1," + ws() + \
        b'"PP"' + ws() + b":" + ws() + b"["
    out, spans = bytearray(head), []
    for i, m in enumerate(members):
        out += ws()
        spans.append((len(out), len(m)))
        out += m + ws()
        if i + 1 < len(members):
            out += b","
    out += ws() + b"]" + ws() + b"}"
    return bytes(out), spans


# ---- logical packets in both forms ----------------------------------------------------------------------------------
def random_logical(rng, world: World, n):
    """[(kind, fields)]: kind 34 or 35 with the fields of a BatchedAcceptReply / BatchedCommit (slots already in the
    TreeMap / TreeSet form both codecs write), plus unknown names and stale versions"""
    out = []
    gids = list(world.groups)
    for _ in range(n):
        gid = int(rng.choice(gids))
        name, ver, members = world.groups[gid]
        u = int(rng.integers(0, 20))
        if u == 0:
            name = name[:-1] + ("?" if name[-1] != "?" else "!")
        elif u == 1:
            ver += 1
        base = int(rng.choice([0, (1 << 31) - 3, -5]))
        if rng.integers(0, 2):
            m = {}
            for s in rng.integers(0, 12, size=int(rng.integers(0, 9))):
                m[wrap32(base + int(s))] = int(rng.integers(-(1 << 62), 1 << 62))
            slots = sorted(m)
            out.append((34, dict(name=name, ver=ver, acc=int(rng.choice(members + [77])), bnum=int(rng.integers(-2**31, 2**31)),
                                 coord=int(rng.choice(members)), first=slots[0] if slots else 0,
                                 cp=int(rng.integers(-2**31, 2**31)), rid=m[slots[0]] if slots else 0, slots=slots,
                                 rids=[m[s] for s in slots])))
        else:
            slots = sorted(set(wrap32(base + int(s)) for s in rng.integers(0, 12, size=int(rng.integers(0, 9)))))
            out.append((35, dict(name=name, ver=ver, bnum=int(rng.integers(-2**31, 2**31)), coord=int(rng.choice(members)),
                                 med=int(rng.integers(-2**31, 2**31)), slots=slots, group=members)))
    return out


def as_bytes(kind, f):
    if kind == 34:
        return wire.encode_batched_accept_reply(f["name"], f["ver"], f["acc"], f["bnum"], f["coord"], f["first"], f["cp"],
                                                f["rid"], f["slots"], f["rids"])
    return wire.encode_batched_commit(f["name"], f["ver"], f["bnum"], f["coord"], f["med"], f["slots"], f["group"])


def as_json(kind, f, rng=None):
    if kind == 34:
        b = pj.batched_accept_reply_json(f["name"], f["ver"], f["acc"], f["bnum"], f["coord"], f["first"], f["cp"],
                                         f["rid"], f["slots"], f["rids"])
    else:
        b = pj.batched_commit_json(f["name"], f["ver"], f["bnum"], f["coord"], f["med"], f["slots"], f["group"])
    if rng is None:
        return b
    return dumps_var(json.loads(b.decode("iso-8859-1")), rng)


def group_into_packets(rng, members):
    """member JSON bytes -> (packets, [(packet index, offset in packet, length)] per member in order): some bare, the
    rest in wrappers of random sizes, some with whitespace"""
    pkts, spans = [], []
    i = 0
    while i < len(members):
        if rng.integers(0, 4) == 0:
            pkts.append(members[i])
            spans.append((len(pkts) - 1, 0, len(members[i])))
            i += 1
            continue
        k = int(rng.integers(1, 12))
        w, sp = wrap(members[i: i + k], rng if rng.integers(0, 2) else None)
        pkts.append(w)
        spans += [(len(pkts) - 1, o, l) for o, l in sp]
        i += k
    return pkts, spans


# ---- the schema, restated -----------------------------------------------------------------------------------------
class Bad(Exception):
    pass


class FloatVal:
    """a number with a fraction or an exponent: fine where a value is skipped, malformed where an int is read"""

    def __init__(self, s):
        self.s = s


def _strict_loads(b: bytes):
    def no_float(s):
        return FloatVal(s)

    def no_const(s):
        raise Bad("constant")

    def pairs(kv):
        return dict(kv)  # the last duplicate wins
    try:
        return json.loads(b.decode("iso-8859-1"), parse_float=no_float, parse_constant=no_const,
                          object_pairs_hook=pairs)
    except (ValueError, RecursionError) as e:
        raise Bad(str(e))


def _int(d, k, bits=32):
    v = d.get(k, None)
    if type(v) is not int or not -(1 << (bits - 1)) <= v < (1 << (bits - 1)):
        raise Bad(k)
    return v


def _ballot(d):
    v = d.get("B")
    if not isinstance(v, str) or v.count(":") != 1:
        raise Bad("B")
    out = []
    for part in v.split(":"):
        t = part[1:] if part.startswith("-") else part
        if not t.isdigit() or not t.isascii() or (len(t) > 1 and t[0] == "0"):
            raise Bad("B")
        x = int(part)
        if not -(1 << 31) <= x < (1 << 31):
            raise Bad("B")
        out.append(x)
    return out


def model_member(world: World, d, node):
    """(status, replies [tuples], decisions [tuples]) of one member object; raises Bad on a schema failure"""
    if not isinstance(d, dict):
        raise Bad("member not an object")
    if _int(d, "type") != 90:
        raise Bad("type")
    pt = _int(d, "PT")
    if pt != 37 and not isinstance(d.get("ID"), str):
        raise Bad("ID")
    ver = _int(d, "V")
    reply = pt in (8, 34)
    if reply:
        sndr, slot, cp, qid = _int(d, "SNDR"), _int(d, "S"), _int(d, "CP_S"), _int(d, "QID", 64)
        bn, bc = _ballot(d)
        nack = d.get("NACK", False)
        if not isinstance(nack, bool):
            raise Bad("NACK")
        if pt == 34:
            sl = d.get("SLOTS")
            if not isinstance(sl, list) or len(sl) % 2:
                raise Bad("SLOTS")
            for i, x in enumerate(sl):
                if type(x) is not int or not -(1 << (31 if i % 2 == 0 else 63)) <= x < (1 << (31 if i % 2 == 0 else 63)):
                    raise Bad("SLOTS")
    elif pt == 35:
        bn, bc = _ballot(d)
        gc = _int(d, "GC_S")
        for key in ("GROUP", "SLOTS"):
            sl = d.get(key)
            if not isinstance(sl, list) or any(type(x) is not int or not -(1 << 31) <= x < (1 << 31) for x in sl):
                raise Bad(key)
    if not (reply or pt == 35) or (pt == 8 and nack):
        return abi.WS_UNHANDLED, [], []
    name = d["ID"]
    if len(name) > 127 or any(ord(c) > 0xFF for c in name):
        return abi.WS_UNKNOWN_NAME, [], []
    gid = world.by_name.get(name)
    if gid is None:
        return abi.WS_UNKNOWN_NAME, [], []
    if world.groups[gid][1] != ver:
        return abi.WS_VERSION, [], []
    members = world.groups[gid][2]
    if reply:
        dst = node if pt == 8 else bc
        if sndr not in members or (pt == 34 and bc not in members):
            return abi.WS_MALFORMED, [], []
        if dst not in members or world.lane_of(dst) is None:
            return abi.WS_NOT_LOCAL, [], []
        who = abi.who(members.index(sndr), members.index(dst), 0)
        if pt == 8:
            q32 = ((qid + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)
            return abi.WS_OK, [(gid, slot, bn, bc, cp, who, q32)], []
        sl = d["SLOTS"]
        return abi.WS_OK, [(gid, sl[i], bn, bc, cp, who, sl[i + 1]) for i in range(0, len(sl), 2)], []
    mask = world.lane_mask(gid)
    if mask == 0:
        return abi.WS_NOT_LOCAL, [], []
    return abi.WS_OK, [], [(gid, s, bn, bc, gc, abi.F_DECISION, mask, 0) for s in d["SLOTS"]]


def model_packet(world: World, b: bytes, node):
    """(status, [member statuses], replies, decisions) the decoder must give one packet (records in member order)"""
    if b.lstrip(b" \t\r\n")[:1] != b"{":
        return abi.WS_UNHANDLED, [], [], []
    try:
        d = _strict_loads(b)
        if not isinstance(d, dict) or _int(d, "type") != 90:
            raise Bad("type")
        pt = _int(d, "PT")
        if pt == 37:
            if "ID" in d or _int(d, "V") != -1 or not isinstance(d.get("PP"), list):
                raise Bad("wrapper")
            objs = d["PP"]
        elif pt in (8, 34, 35):
            objs = [d]
        else:
            return abi.WS_UNHANDLED, [], [], []
        got = [model_member(world, o, node) for o in objs]
    except Bad:
        return abi.WS_MALFORMED, [], [], []
    return abi.WS_OK, [g[0] for g in got], [r for g in got for r in g[1]], [x for g in got for x in g[2]]


def model_batch(world: World, pkts, nodes):
    """(statuses, member statuses, replies, decisions) of a batch: records grouped by gid, batch order within"""
    st, ms, reps, decs = [], [], [], []
    for b, node in zip(pkts, nodes):
        s, m, r, d = model_packet(world, b, node)
        st.append(s)
        ms += m
        reps += r
        decs += d
    reps.sort(key=lambda t: t[0])
    decs.sort(key=lambda t: t[0])
    return st, ms, np.array(reps, dtype=abi.reply_dtype), np.array(decs, dtype=abi.decision_dtype)


def malformed_corpus(world: World):
    """[(packet bytes, receiving node)] with every rule of the schema broken somewhere; the model says the outcome"""
    gid0 = min(g for g, (_, _, m) in world.groups.items() if world.lane_of(m[0]) is not None and
               world.lane_of(m[-1]) is not None)
    name, ver, members = world.groups[gid0]
    rep = pj.batched_accept_reply_json(name, ver, members[0], 3, members[-1], 5, 4, 9, [5, 6], [9, 10])
    com = pj.batched_commit_json(name, ver, 3, members[0], 2, [1, 2], members)
    one = pj.accept_reply_json(name, ver, members[0], 3, members[-1], 5, 4, 9)
    good, _ = wrap([rep, com, one])
    out = [good[:i] for i in range(len(good))]  # every truncation prefix
    sub = lambda b, a, z: b.replace(a, z, 1)
    more = [
        good + b" ",  # trailing whitespace: fine
        good + b"x", good + b"{}", b"  " + good,  # trailing bytes / leading whitespace
        sub(good, b'"ID":"', b'"ID":"\\"'), sub(good, b'"ID":"', b'"ID":"\\\\'),  # escaped quote and backslash run
        sub(good, b'"ID":"', b'"ID":"\\q'), sub(good, b'"ID":"', b'"ID":"\\u12G4'),  # bad escapes
        sub(good, b'"ID":"', b'"ID":"\x01'),  # raw control character
        sub(good, b"[5,", b"{5,"), sub(good, b"]}", b"}]"), sub(good, b"]}", b"]}]"), sub(good, b'"PP":[', b'"PP":[['),
        sub(good, b'"S":5', b'"S":2147483648'), sub(good, b'"S":5', b'"S":-2147483648'),
        sub(good, b'"S":5', b'"S":5.0'), sub(good, b'"S":5', b'"S":5e0'), sub(good, b'"S":5', b'"S":05'),
        sub(good, b'"S":5', b'"S":+5'), sub(good, b'"S":5', b'"S":-0'), sub(good, b'"QID":9', b'"QID":9223372036854775807'),
        sub(good, b'"QID":9', b'"QID":9223372036854775808'), sub(good, b'"QID":9', b'"QID":-9223372036854775808'),
        sub(good, b'"CP_S":4,', b""), sub(good, b'"S":5', b'"S":"5"'), sub(good, b'"B":"3:', b'"B":"+3:'),
        sub(good, b'"B":"3:', b'"B":"03:'), sub(good, b'"B":"3:', b'"B":"-3:'), sub(good, b'"B":"3:', b'"B":3'),
        sub(good, b'"B":"3:', b'"B":"3:-'), sub(good, b'"B":"3:', b'"B":"\\u0033:'),
        sub(good, b"[5,9,6,10]", b"[5,9,6]"), sub(good, b"[5,9,6,10]", b"[]"), sub(good, b'"GROUP":[', b'"GROUP":["x",'),
        sub(good, b'"V":-1', b'"V":0'), sub(good, b'"type":90', b'"type":91'), sub(good, b'"PT":37', b'"PT":36'),
        sub(good, b'"PT":37', b'"PT":37,"ID":"x"'), sub(good, b'"PP":[', b'"PP":5,"Q":['),
        wrap([])[0], b'{"type":90,"PT":37,"V":-1,"PP":[ \n ]}', b'{"type":90,"PT":37,"V":-1,"PP":[1]}',
        wrap([good])[0],  # a nested 37
        b'{"type":90,"PT":37,"V":-1,"PP":[{"type":90,"PT":37,"V":0}]}',  # the shortest valid member: a nested 37
        b'{"type":90,"PT":37,"V":-1,"PP":[{"type":90,"PT":37,"V":0},{"type":90,"PT":37,"V":0}]}',
        b'{"type":90,"PT":37,"V":-1,"PP":[{"type":90,"PT":3,"V":0}]}',  # shorter than any valid member
        wrap([sub(one, b'"QID":9', b'"QID":9,"NACK":true')])[0], wrap([sub(one, b'"QID":9', b'"QID":9,"NACK":false')])[0],
        wrap([sub(one, b'"QID":9', b'"QID":9,"NACK":1')])[0],
        wrap([sub(rep, name.encode("iso-8859-1"), b"x" * 128)])[0], wrap([sub(rep, b'"ID":"', b'"ID":"\\u0100')])[0],
        wrap([sub(rep, b'"SNDR":%d' % members[0], b'"SNDR":77')])[0],
        b'{"type":90,"PT":3,"ID":"a","V":0}', b'{"type":90,"PT":3,"ID":"a","V":0,"PP":[1,]}', b'[1]', b"", b"   ",
        b'{"type":90,"PT":35,"ID":' + _jstr(name) + b',"V":%d,"B":"1:2","GC_S":0,"GROUP":[],"SLOTS":[1],"PP":[{"a":[[[]]]}]}' % ver,
        wrap([rep, com], None)[0].replace(b",", b" , ", 3),
    ]
    return [(p, members[0]) for p in out + more]
