"""Cases and a model shared by tests/test_wire_client.py (k_json_client on the host, tests/emu/wire_client_emu.cpp) and
tests/test_wire_client_gpu.py (the same call through the C ABI): a client's own REQUEST packets, bare JSON objects in
the org.json form a client writes and the json-smart form, with and without the receiver's address stamps, and the
connection each came in on.

The model reads a packet as the reference does: RequestPacket(JSONObject) :512-567 takes "CA" when present, else the
sender stamp MessageExtractor.stampAddressIntoJSONObject :348-376 put there (it never overwrites one), which is the
connection's remote address; "LA" likewise with the receiver stamp and the local address.  A BATCH entry is built from
its own object (:541-552), which nobody stamps.  The resolved request then decodes as wire_coord_cases.expected_requests
says for its byte form."""
from __future__ import annotations

import json

import numpy as np

from gigapaxos_b200 import abi, packets_json as pj, wire
from wire_coord_cases import expected_requests, random_request
from wire_dev_cases import World
from wire_fwd_cases import json_string, model_fields, wrapper

WS = b" \t\n\r"
CONNS = [("10.1.2.3", 40001), ("192.168.0.7", 65535), ("1.0.0.1", 1), ("172.16.5.4", 2000)]
LISTENS = [("10.0.0.9", 2000), ("10.0.0.10", 2001)]


def peer_rows(peers):
    """[(sender, receiver)] -> abi.wire_peer_dtype rows (at least one)"""
    return wire.wire_peers(list(peers) or [(None, None)])


# ---- writing packets -------------------------------------------------------------------------------------------------
def obj_bytes(d: dict, rng) -> bytes:
    """d as compact JSON with every QV (at any depth) written by json_string: raw, escaped or \\u00XX"""
    vals = []

    def mark(o):
        if isinstance(o, dict):
            for k in list(o):
                if k == "QV" and isinstance(o[k], str):
                    vals.append(o[k].encode("iso-8859-1"))
                    o[k] = "\0QV%d" % (len(vals) - 1)
                else:
                    mark(o[k])
        elif isinstance(o, list):
            for x in o:
                mark(x)
    d = json.loads(json.dumps(d))
    mark(d)
    b = json.dumps(d, separators=(",", ":")).encode("ascii")
    for k, v in enumerate(vals):
        b = b.replace(b'"\\u0000QV%d"' % k, json_string(v, rng), 1)
    return b


def client_obj(r: wire.Request, smart: bool) -> dict:
    """the object a client writes for r: org.json's toJSONObjectImpl keys or json-smart's"""
    return pj._request_smart(r, pj.PT_REQUEST) if smart else pj._request_org(r, pj.PT_REQUEST)


def stamp(d: dict, sender, receiver, form: str) -> dict:
    """the receiver's stamps: form "org" ("a.b.c.d:port" and the deprecated _SNDR_IP / _SNDR_PORT), "smart"
    ("/a.b.c.d:port") or "host" ("host.name/a.b.c.d:port", InetSocketAddress.toString() of a resolved address)"""
    d = dict(d)
    pre = {"org": "", "smart": "/", "host": "client.example/"}[form]
    if sender is not None:
        d.setdefault("_SNDR_ADDRESS", f"{pre}{sender[0]}:{sender[1]}")
        if form == "org":
            d.setdefault("_SNDR_IP", sender[0])
            d.setdefault("_SNDR_PORT", int(sender[1]))
    if receiver is not None:
        d.setdefault("_RCVR_ADDRESS", f"{pre}{receiver[0]}:{receiver[1]}")
    return d


# ---- the model -------------------------------------------------------------------------------------------------------
def _i32(v):
    return type(v) is int and -(1 << 31) <= v < (1 << 31)


def _addr(s):
    t = s.rsplit("/", 1)[-1]
    ip, port = t.rsplit(":", 1)
    return (ip, int(port))


def resolve(d: dict, peer, top: bool):
    """(d with the resolved "CA" / "LA" written in, whether a fallback port was unknown).  peer = (sender, receiver) or
    None: no fallback"""
    d = dict(d)
    unknown = False
    for key, st, k in (("CA", "_SNDR_ADDRESS", 0), ("LA", "_RCVR_ADDRESS", 1)):
        if key in d:
            continue
        if st in d:
            d[key] = d[st]
        elif top and peer is not None:
            a = peer[k]
            if a is None or not a[1]:
                unknown = True
            else:
                d[key] = f"/{a[0]}:{a[1]}"
    if top and isinstance(d.get("BATCH"), list):
        d["BATCH"] = [resolve(x, None, False)[0] if isinstance(x, dict) else x for x in d["BATCH"]]
    return d, unknown


def as_request(d: dict) -> wire.Request:
    """the wire.Request of a resolved request object that model_fields accepts"""
    return wire.Request(d["ID"] if "ID" in d else "", d.get("V", 0), d["QID"], d["QV"].encode("iso-8859-1"),
                        stop=d.get("STOP", False), entry_replica=d["E"], entry_time=d["ET"],
                        client=_addr(d["CA"]) if "CA" in d else None, listen=_addr(d["LA"]) if "LA" in d else None,
                        should_return=d.get("QF", False), forward_count=d.get("NFWDS", 0),
                        broadcasted=d.get("BC", False),
                        batched=tuple(as_request(dict(x, ID=d["ID"], V=d["V"])) for x in d.get("BATCH", [])))


def model_packet(b: bytes, peer):
    """(status, None) for a packet the call must not decode, else (None, the resolved wire.Request): its status and
    records are the byte decoder's (expected_requests)"""
    s = b.lstrip(WS)
    if not s.startswith(b"{"):
        return abi.WS_UNHANDLED, None
    try:
        d = json.loads(b.decode("iso-8859-1"), parse_constant=lambda c: (_ for _ in ()).throw(ValueError(c)))
    except ValueError:
        return abi.WS_MALFORMED, None
    if type(d) is not dict or not _i32(d.get("type")):
        return abi.WS_MALFORMED, None
    if d["type"] != pj.PT_PAXOS_PACKET:
        return abi.WS_UNHANDLED, None
    if not _i32(d.get("PT")):
        return abi.WS_MALFORMED, None
    if d["PT"] != pj.PT_REQUEST:
        return abi.WS_UNHANDLED, None
    if type(d.get("ID")) is not str or not _i32(d.get("V")):
        return abi.WS_MALFORMED, None
    r, unknown = resolve(d, peer, True)
    st = model_fields(r, True)
    if st == abi.WS_OK and unknown:
        st = abi.WS_UNHANDLED
    return (st, None) if st != abi.WS_OK else (None, as_request(r))


def expected(world: World, pkts, peers):
    """(status, reqs, meta, payload) the call must give for [(bytes, node)] and peers [(sender, receiver)] (None: the
    call is given none), byte for byte"""
    models = [model_packet(b, None if peers is None else peers[k]) for k, (b, _) in enumerate(pkts)]
    est, reqs, meta, _ = expected_requests(world, [(b, node, m[1]) for (b, node), m in zip(pkts, models)])
    status = [m[0] if m[1] is None else s for m, s in zip(models, est)]
    # payload: each OK packet's values in packet order, each padded to 16; records sorted stably by gid
    pay, offs = bytearray(), []
    for k, (m, s) in enumerate(zip(models, status)):
        if s != abi.WS_OK:
            continue
        gid = world.by_name[m[1].paxos_id]
        for q in [m[1]] + list(m[1].batched):
            offs.append((gid, len(pay)))
            pay += q.value + bytes(-len(q.value) % 16)
    offs.sort(key=lambda t: t[0])
    reqs = reqs.copy()
    if len(reqs):
        reqs["payload_off"] = [o for _, o in offs]
    return np.array(status, np.int32), reqs, meta, np.frombuffer(bytes(pay), np.uint8)


# ---- random traffic --------------------------------------------------------------------------------------------------
def random_client_packets(rng, world: World, n, mixed=True):
    """([(bytes, node)], [(sender, receiver)]): RequestPackets as clients send them (no "CA" mostly, entryReplica -1
    often), org.json or json-smart, stamped or not, over connections with known and unknown ports, at local and
    non-local nodes; mixed: also byteified REQUESTs, wrappers and other JSON"""
    from wire_coord_cases import random_request_packets
    out, peers = [], []
    for b, node, req in random_request_packets(rng, world, n):
        u = int(rng.integers(0, 20))
        if mixed and u == 0:
            out.append((b, node))  # the byte form
        elif mixed and u == 1:
            out.append((wrapper([pj.request_json(req)]), node))
        elif mixed and u == 2:
            out.append((b'{"type":3,"x":[1,{"y":null}]}', node))  # another JSON packet type
        else:
            if rng.integers(0, 4):  # a client's own request: no clientAddress, usually no listenAddress
                req.client = None
                req.listen = None if rng.integers(0, 4) else req.listen
            d = client_obj(req, bool(rng.integers(0, 2)))
            if rng.integers(0, 3) == 0:
                d = stamp(d, CONNS[int(rng.integers(0, len(CONNS)))] if rng.integers(0, 4) else None,
                          LISTENS[int(rng.integers(0, 2))] if rng.integers(0, 4) else None,
                          ("org", "smart", "host")[int(rng.integers(0, 3))])
            lead = WS[: int(rng.integers(0, 3))] if rng.integers(0, 8) == 0 else b""
            out.append((lead + obj_bytes(d, rng), node))
        snd = CONNS[int(rng.integers(0, len(CONNS)))] if rng.integers(0, 15) else (CONNS[0][0], 0)
        rcv = LISTENS[int(rng.integers(0, 2))] if rng.integers(0, 20) else None
        peers.append((snd, rcv))
    return out, peers


def random_resolvable(rng, world: World, n):
    """([(bytes, node)], peers, [(bytes, node)] the same requests with the resolved "CA" / "LA" written out): JSON client
    requests whose every fallback port is known, for the comparison with gpx_wire_decode_json_requests_device"""
    pkts, inserted, peers = [], [], []
    gids = list(world.groups)
    for _ in range(n):
        gid = int(rng.choice(gids))
        name, ver, members = world.groups[gid]
        req = random_request(rng, name, ver, batched=0 if rng.integers(0, 2) else int(rng.integers(1, 6)))
        req.client = None if rng.integers(0, 4) else req.client
        local = [m for m in members if m in world.lanes]
        node = int(rng.choice(local)) if local and rng.integers(0, 8) else int(rng.choice(world.lanes + [7]))
        d = client_obj(req, bool(rng.integers(0, 2)))
        if rng.integers(0, 3) == 0:
            d = stamp(d, CONNS[int(rng.integers(0, len(CONNS)))], LISTENS[int(rng.integers(0, 2))],
                      ("org", "smart", "host")[int(rng.integers(0, 3))])
        peer = (CONNS[int(rng.integers(0, len(CONNS)))], LISTENS[int(rng.integers(0, 2))])
        r, _ = resolve(d, peer, True)
        seed = int(rng.integers(1 << 30))
        pkts.append((obj_bytes(d, np.random.default_rng(seed)), node))
        inserted.append((obj_bytes(r, np.random.default_rng(seed)), node))
        peers.append(peer)
    return pkts, peers, inserted


# ---- the corpus ------------------------------------------------------------------------------------------------------
def corpus(world: World):
    """[(bytes, node, peer, expected status, expected (client, listen) of the outer request or None)], one rule each"""
    gid = min(g for g in world.groups if any(m in world.lanes for m in world.groups[g][2]))
    name, ver, members = world.groups[gid]
    node = next(m for m in members if m in world.lanes)
    conn, lis = ("10.1.2.3", 40001), ("10.0.0.9", 2000)
    peer = (conn, lis)
    base = wire.Request(name, ver, 5, b"x/y\"z\x01\xe9", entry_replica=-1, entry_time=77)
    org = json.loads(pj.client_request_json(base).decode("iso-8859-1"))
    sub = wire.Request(name, ver, 6, b"b")

    def pk(d, **kw):
        d = dict(d)
        for k, x in kw.items():
            if x is KeyError:
                d.pop(k, None)
            else:
                d[k] = x
        return json.dumps(d, separators=(",", ":")).encode("iso-8859-1")
    OK, UN, MAL = abi.WS_OK, abi.WS_UNHANDLED, abi.WS_MALFORMED
    c = [
        # the org.json bytes a client writes, as they are; no address key: the connection's
        (pj.client_request_json(base), node, peer, OK, (conn, lis)),
        (pj.client_request_json(base, smart=True), node, peer, OK, (conn, lis)),
        (b" \n\t" + pj.client_request_json(base), node, peer, OK, (conn, lis)),
        # a stamp in each form beats the connection
        (pj.client_request_json(base, ("1.2.3.4", 5), ("5.6.7.8", 9)), node, peer, OK, (("1.2.3.4", 5), ("5.6.7.8", 9))),
        (pj.client_request_json(base, ("1.2.3.4", 5), ("5.6.7.8", 9), smart=True), node, peer, OK,
         (("1.2.3.4", 5), ("5.6.7.8", 9))),
        (pk(org, _SNDR_ADDRESS="c.example/1.2.3.4:5"), node, peer, OK, (("1.2.3.4", 5), lis)),
        (pk(org, _RCVR_ADDRESS="5.6.7.8:9"), node, peer, OK, (conn, ("5.6.7.8", 9))),
        # a "CA" / "LA" beats both
        (pk(org, CA="/9.9.9.9:99", _SNDR_ADDRESS="1.2.3.4:5"), node, peer, OK, (("9.9.9.9", 99), lis)),
        (pk(org, LA="/8.8.8.8:88", _RCVR_ADDRESS="5.6.7.8:9"), node, peer, OK, (conn, ("8.8.8.8", 88))),
        # no peers given: an absent address is all zeros
        (pj.client_request_json(base), node, None, OK, (None, None)),
        (pk(org, _SNDR_ADDRESS="1.2.3.4:5"), node, None, OK, (("1.2.3.4", 5), None)),
        # port 0, IPv6, a hostname in each position: the host's
        (pj.client_request_json(base), node, ((conn[0], 0), lis), UN, None),
        (pj.client_request_json(base), node, (conn, None), UN, None),
        (pk(org, CA="/[::1]:80"), node, peer, UN, None),
        (pk(org, CA="host.example:80"), node, peer, UN, None),
        (pk(org, CA="/1.2.3.4:0"), node, peer, UN, None),
        (pk(org, LA="/[::1]:80"), node, peer, UN, None),
        (pk(org, _SNDR_ADDRESS="[::1]:80"), node, peer, UN, None),
        (pk(org, _SNDR_ADDRESS="host.example:80"), node, peer, UN, None),
        (pk(org, _SNDR_ADDRESS="1.2.3.4:0"), node, peer, UN, None),
        (pk(org, _RCVR_ADDRESS="0:0:0:0:0:0:0:1:2000"), node, peer, UN, None),
        (pk(org, _RCVR_ADDRESS="me.example:2000"), node, peer, UN, None),
        (pk(org, _SNDR_ADDRESS=5), node, peer, MAL, None),  # not a string, as for "CA"
        # a key that only starts like a stamp is skipped
        (pk(org, _SNDR_ADDRESX="1.2.3.4:5", _SNDR_ADDRES="1.2.3.4:5", _SNDR_ADDRESS_="1.2.3.4:5"), node, peer, OK,
         (conn, lis)),
        (pj.client_request_json(base).replace(b"{", b'{"_SNDR_\\u0041DDRESS":"1.2.3.4:5",', 1), node, peer, OK,
         (("1.2.3.4", 5), lis)),
        # BATCH entries take their own "CA", else their own stamp, else nothing: never the connection
        (pk(org, BATCH=[pj._request_org(sub, 1), dict(pj._request_org(sub, 1), CA="/7.7.7.7:7"),
                        dict(pj._request_org(sub, 1), _SNDR_ADDRESS="6.6.6.6:6")]), node, peer, OK, (conn, lis)),
        (pk(org, BATCH=[dict(pj._request_org(sub, 1), _SNDR_ADDRESS="[::1]:6")]), node, peer, UN, None),
        (pk(org, BATCH=[dict(pj._request_org(sub, 1), BATCH=[])]), node, peer, MAL, None),
        # other forms: the byte form, a wrapper, other JSON types -- the host's
        (wire.encode_request(base), node, peer, UN, None),
        (wrapper([pj.request_json(base)]), node, peer, UN, None),
        (pk(org, PT=3), node, peer, UN, None),
        (b'{"type":5,"x":1}', node, peer, UN, None),
        (b'{"type":5}', node, peer, UN, None),
        (b"", node, peer, UN, None),
        (b"   ", node, peer, UN, None),
        (b"[1]", node, peer, UN, None),
        # names, versions, the receiving node
        (pk(org, ID=name + "?"), node, peer, abi.WS_UNKNOWN_NAME, None),
        (pk(org, V=ver + 1), node, peer, abi.WS_VERSION, None),
        (pj.client_request_json(base), 7, peer, abi.WS_NOT_LOCAL, None),
        # malformed JSON and schema failures
        (pj.client_request_json(base)[:-1], node, peer, MAL, None),
        (pj.client_request_json(base) + b"x", node, peer, MAL, None),
        (b"{", node, peer, MAL, None),
        (pk(org, type=KeyError), node, peer, MAL, None),
        (pk(org, type="90"), node, peer, MAL, None),
        (pk(org, PT=KeyError), node, peer, MAL, None),
        (pk(org, ID=KeyError), node, peer, MAL, None),
        (pk(org, V=KeyError), node, peer, MAL, None),
        (pk(org, QID=KeyError), node, peer, MAL, None),
        (pk(org, E=1.5), node, peer, MAL, None),
        (pk(org, RV="r"), node, peer, UN, None),
        (pk(org, DIG="d"), node, peer, UN, None),
        (pk(org, QV="xĀ"), node, peer, UN, None),
    ]
    return c


def bulk_client_packets(n, G, rng, value_len=1):
    """n org.json client packets of one request of value_len bytes each (bench.py cfg2's requests: groups
    NoopPaxosApp<g>, no "CA"), the same packets with their connection's addresses written out as "CA" / "LA", and the
    peers (abi.wire_peer_dtype): clients 10.9.8.x on ports 1024-65535, all received on 10.0.0.1:2000.  n <= G: one
    packet per group, in a random order."""
    gid = rng.permutation(G)[:n] if n <= G else rng.integers(0, G, size=n)
    port = rng.integers(1024, 65536, size=n)
    ip3 = rng.integers(1, 255, size=n)
    qid = rng.integers(1, 1 << 62, size=n)
    val = bytes(rng.integers(97, 123, size=value_len, dtype=np.uint8))
    plain, inserted = [], []
    for k in range(n):
        head = b'{"type":90,"PT":1,"ID":"NoopPaxosApp%d","V":0,"QID":%d,"QV":"%s","ET":1700000000000,"E":-1' % (
            gid[k], qid[k], val)
        plain.append(head + b"}")
        inserted.append(head + b',"CA":"/10.9.8.%d:%d","LA":"/10.0.0.1:2000"}' % (ip3[k], port[k]))
    peers = np.zeros(n, abi.wire_peer_dtype)
    peers["sender_ip"] = np.stack([np.full(n, 10), np.full(n, 9), np.full(n, 8), ip3], axis=1)
    peers["sender_port"] = port
    peers["receiver_ip"] = [10, 0, 0, 1]
    peers["receiver_port"] = 2000
    return plain, inserted, peers
