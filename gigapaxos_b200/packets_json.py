"""The inter-replica packets the reference sends STRINGIFIED, and the cross-group packet batcher (SURVEY.md 8a row a14).

Four packet types travel byteified (REQUEST, ACCEPT, BATCHED_ACCEPT_REPLY, BATCHED_COMMIT: include/gpx_wire.h,
paxosutil/PaxosMessenger.java:126-132, paxosutil/PaxosPacketDemultiplexerFast.java:82-95); everything else a gpx-backed
node exchanges with a Java peer is the JSON string of PaxosPacket.toJSONObject() (paxospackets/PaxosPacket.java:478-494:
{"type": 90, "PT": <type>, "ID": paxosID, "V": version} + the subclass's toJSONObjectImpl()).  Node ids are integers
(IntegerMap.allInt(), which byteification requires as well: PaxosMessenger.java:127, :187).  This module holds the ones
the phase-2 path produces besides the DECISION / PREPARE forms of journal.py:

  ACCEPT_REPLY (8), singleton   a NACK (higher ballot) or an undigest request is never coalesced into a
                                BatchedAcceptReply (PaxosPacketBatcher.allPositiveAcceptReplies :423-430); AcceptReplyPacket
                                .toJSONObjectImpl :196-206
  BATCHED_ACCEPT (36)           digest mode: the coordinator's ACCEPTs of one (paxosID, ballot) as slot -> digest and
                                slot -> requestID maps; BatchedAccept.toJSONObjectImpl :99-146, merge rule addBatchedAccept
                                :194-209 (wrap-aware max of medianCheckpointedSlot, TreeMap.putAll)
  PREPARE (2), PREPARE_REPLY (7)  phase 1 between nodes.  A PREPARE_REPLY carries the acceptor's accepted pvalues as full
                                PValuePacket JSON objects incl. the request values (PrepareReplyPacket.toJSONObjectImpl
                                :131-143, addAcceptedToJSON :191-199); on the engine side it is gpx_prepare_reply_rec
                                records (continued with GPX_F_MORE past GPX_MAX_WINDOW pvalues, the analogue of
                                PrepareReplyPacket.fragment :231-258) + the request bodies in a payload arena -- the
                                input of gpx_handle_prepare_replies.
  SYNC_DECISIONS (32)           a replica asks for the decisions it missed (SyncDecisionsPacket.toJSONObjectImpl :79-88); the
                                answer is the missing DECISIONs as full PValuePackets.  serve_sync_request looks them up
                                with gpx_log_find + gpx_log_gather at the donor (PISM.handleSyncDecisionsPacket :2426-2510,
                                getActualDecisions :2539-2583); decisions_to_records makes them replayable at the requester.
  BATCHED_PAXOS_PACKET (37)     PaxosPacketBatcher.batch :280-303: the messaging tasks of one batcher sweep grouped by
                                recipient set (first-seen order: LinkedHashMap), each group's packets in one
                                {"PP": [...]} wrapper; BatchedPaxosPacket.toJSONObjectImpl :77-84.  process() :270-277 does
                                this only when BATCH_ACROSS_GROUPS and more than MIN_PP_BATCH_SIZE (3) tasks are pending;
                                the receiver unwraps (PaxosManager.java:1087-1090).

Key order inside a JSON object is not significant (org.json / json-smart objects are hash maps).
"""
from __future__ import annotations

import json
from typing import Dict, Iterable, List, Sequence, Tuple, Union

PT_REQUEST, PT_PREPARE, PT_ACCEPT, PT_DECISION, PT_PREPARE_REPLY, PT_ACCEPT_REPLY = 1, 2, 3, 6, 7, 8
PT_SYNC_DECISIONS, PT_BATCHED_ACCEPT, PT_BATCHED_PAXOS_PACKET, PT_PAXOS_PACKET = 32, 36, 37, 90  # PaxosPacketType :202-291
PT_BATCHED_ACCEPT_REPLY, PT_BATCHED_COMMIT = 34, 35
CHARSET = "iso-8859-1"  # PaxosPacket.CHARSET :439, BatchedAccept.CHARSET :36

BATCH_ACROSS_GROUPS = True  # PaxosConfig.java:807
MIN_PP_BATCH_SIZE = 3  # PaxosConfig.java:860


def _dumps(d: dict) -> bytes:
    """Strings leave a Java node as String.getBytes("ISO-8859-1") (nio/MessageNIOTransport.java:524, JSONMessenger.java:463;
    the journal: SQLPaxosLogger.java:1094, CHARSET :1313).  Every non-ASCII character is written as a \\uXXXX escape here,
    so the bytes are the same under any charset and every JSON parser reads back the same characters; frames a Java node
    wrote may hold raw ISO-8859-1 bytes, so the reading side decodes with that charset."""
    return json.dumps(d, separators=(",", ":")).encode("ascii")


def _loads(b: bytes) -> dict:
    return json.loads(b.decode(CHARSET))


def _base(pt: int, paxos_id, version: int) -> dict:
    d = {"type": PT_PAXOS_PACKET, "PT": pt}
    if paxos_id is not None:  # JSONObject.put(key, null) removes the key
        d["ID"] = paxos_id
    d["V"] = int(version)
    return d


def _i32(x: int) -> int:
    return ((int(x) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


# ---- ACCEPT_REPLY ---------------------------------------------------------------------------------------------------
def accept_reply_json(paxos_id: str, version: int, acceptor: int, bnum: int, bcoord: int, slot_number: int,
                      max_checkpointed_slot: int, request_id: int, undigest_request: bool = False) -> bytes:
    d = _base(PT_ACCEPT_REPLY, paxos_id, version)
    d.update({"SNDR": int(acceptor), "B": f"{int(bnum)}:{int(bcoord)}", "S": int(slot_number),
              "CP_S": int(max_checkpointed_slot), "QID": int(request_id)})
    if undigest_request:
        d["NACK"] = True
    return _dumps(d)


def accept_replies_to_packets(replies, names: Dict[int, Tuple[str, int]], node_of_lane: Sequence[int]) -> List[bytes]:
    """The singleton ACCEPT_REPLYs among engine reply records (abi.reply_dtype): the NACKs, i.e. replies whose ballot is
    above the ACCEPT's own (PISM.handleAccept :1139-1142 answers with the acceptor's ballot).  Positive replies go into
    gpx_wire_encode_batched_accept_reply instead.  names: gid -> (paxosID, version)."""
    from . import abi
    out = []
    for r in replies:
        who = int(r["who"])
        if (who >> 16) & abi.F_VOID or not (who >> 16) & abi.F_NACK:
            continue
        pid, ver = names[int(r["gid"])]
        out.append(accept_reply_json(pid, ver, node_of_lane[who & 0xFF], int(r["bnum"]), int(r["bcoord"]),
                                     int(r["slot"]), int(r["max_cp"]), int(r["req_id"])))
    return out


def batched_accept_reply_json(paxos_id: str, version: int, acceptor: int, bnum: int, bcoord: int, slot_number: int,
                              max_checkpointed_slot: int, request_id: int, slots: Sequence[int],
                              request_ids: Sequence[int]) -> bytes:
    """BatchedAcceptReply.toJSONSmartImpl :86-96 on top of AcceptReplyPacket.toJSONSmartImpl :214-224: the header of the
    first reply and SLOTS = [slot, requestID, ...] in ascending slot order (the TreeMap; a repeated slot keeps its last
    requestID).  Wrapped by batched_paxos_packet_json, this is how a loaded Java peer's replies arrive."""
    m = {}
    for s, q in zip(slots, request_ids):
        m[int(s)] = int(q)
    d = _base(PT_BATCHED_ACCEPT_REPLY, paxos_id, version)
    d.update({"SNDR": int(acceptor), "B": f"{int(bnum)}:{int(bcoord)}", "S": int(slot_number),
              "CP_S": int(max_checkpointed_slot), "QID": int(request_id)})
    d["SLOTS"] = [x for s in sorted(m) for x in (s, m[s])]
    return _dumps(d)


def batched_commit_json(paxos_id: str, version: int, bnum: int, bcoord: int, median_cp: int, slots: Sequence[int],
                        group: Iterable[int]) -> bytes:
    """BatchedCommit.toJSONSmartImpl :140-149: ballot, medianCheckpointedSlot, the group and the slots (a TreeSet:
    ascending, distinct)"""
    d = _base(PT_BATCHED_COMMIT, paxos_id, version)
    d.update({"B": f"{int(bnum)}:{int(bcoord)}", "GC_S": int(median_cp), "GROUP": [int(g) for g in group],
              "SLOTS": sorted(set(int(s) for s in slots))})
    return _dumps(d)


# ---- BATCHED_ACCEPT -------------------------------------------------------------------------------------------------
class BatchedAccept:
    """paxospackets/BatchedAccept.java: the digested ACCEPTs of one (paxosID, version, ballot) to one group"""

    def __init__(self, paxos_id: str, version: int, bnum: int, bcoord: int, median_cp: int, group: Iterable[int]):
        self.paxos_id, self.version, self.bnum, self.bcoord = paxos_id, int(version), int(bnum), int(bcoord)
        self.median_cp = int(median_cp)
        self.group = sorted(set(int(g) for g in group))
        self.slot_digests: Dict[int, bytes] = {}
        self.slot_request_ids: Dict[int, int] = {}

    def add_accept(self, slot: int, digest: bytes, request_id: int, median_cp: int, bnum=None, bcoord=None,
                   paxos_id=None):  # addAccept :229-241
        if (bnum is not None and (int(bnum), int(bcoord)) != (self.bnum, self.bcoord)) or \
                (paxos_id is not None and paxos_id != self.paxos_id):
            raise RuntimeError("Unable to combine accepts of different ballots / groups")
        if _i32(int(median_cp) - self.median_cp) > 0:  # wrap-aware max
            self.median_cp = int(median_cp)
        self.slot_digests[int(slot)] = bytes(digest)
        self.slot_request_ids[int(slot)] = int(request_id)
        return self

    def add_batched_accept(self, other: "BatchedAccept") -> bool:  # addBatchedAccept :194-209
        if (other.bnum, other.bcoord) != (self.bnum, self.bcoord) or other.paxos_id != self.paxos_id:
            raise RuntimeError("Unable to combine batched accepts of different ballots / groups")
        if _i32(other.median_cp - self.median_cp) > 0:
            self.median_cp = other.median_cp
        self.slot_digests.update(other.slot_digests)
        self.slot_request_ids.update(other.slot_request_ids)
        return True

    def slots(self) -> List[int]:  # TreeMap<Integer,..>: natural (signed) order
        return sorted(self.slot_digests)

    def to_json(self) -> bytes:
        d = _base(PT_BATCHED_ACCEPT, self.paxos_id, self.version)
        d.update({"B": f"{self.bnum}:{self.bcoord}", "GC_S": self.median_cp, "GROUP": list(self.group),
                  "S_DIGS": [[s, self.slot_digests[s].decode(CHARSET)] for s in self.slots()],
                  "S_QIDS": [[s, self.slot_request_ids[s]] for s in sorted(self.slot_request_ids)]})
        return _dumps(d)

    @staticmethod
    def from_json(j: Union[bytes, dict]) -> "BatchedAccept":
        if not isinstance(j, dict):
            j = _loads(j)
        assert j["type"] == PT_PAXOS_PACKET and j["PT"] == PT_BATCHED_ACCEPT
        bn, bc = (int(x) for x in j["B"].split(":"))
        b = BatchedAccept(j["ID"], j["V"], bn, bc, j["GC_S"], j["GROUP"])
        for s, dig in j["S_DIGS"]:
            b.slot_digests[int(s)] = dig.encode(CHARSET)
        for s, q in j["S_QIDS"]:
            b.slot_request_ids[int(s)] = int(q)
        return b

    def to_digested_accepts(self, gid: int, sender_lane: int, value_len: int = 0):
        """the engine-side form: one digests.DigestedAccept per slot (PISM.handleBatchedAccept :1183-1210 unrolls a
        BatchedAccept into per-slot ACCEPTs that PendingDigests.match joins with the request bodies)"""
        import numpy as np
        from . import abi
        from .digests import DigestedAccept
        out = []
        for s in self.slots():
            r = np.zeros((), dtype=abi.accept_dtype)
            r["gid"], r["slot"], r["bnum"], r["bcoord"] = gid, s, self.bnum, self.bcoord
            r["median_cp"], r["req_id"], r["nreq"], r["sender"] = self.median_cp, self.slot_request_ids[s], 1, sender_lane
            out.append(DigestedAccept(r, self.slot_digests[s], value_len))
        return out


def batch_digested_accepts(accs, names: Dict[int, Tuple[str, int]], groups: Dict[int, Sequence[int]]) -> List[BatchedAccept]:
    """PaxosPacketBatcher.enqueueImpl(BatchedAccept) :158-173: digested ACCEPTs (digests.DigestedAccept) of a sweep merged
    per (paxosID, ballot), first-seen order"""
    merged: Dict[Tuple[str, int, int], BatchedAccept] = {}
    for a in accs:
        r = a.rec
        pid, ver = names[int(r["gid"])]
        key = (pid, int(r["bnum"]), int(r["bcoord"]))
        if key not in merged:
            merged[key] = BatchedAccept(pid, ver, key[1], key[2], int(r["median_cp"]), groups[int(r["gid"])])
        merged[key].add_accept(int(r["slot"]), a.digest, int(r["req_id"]), int(r["median_cp"]))
    return list(merged.values())


# ---- PREPARE / PREPARE_REPLY ----------------------------------------------------------------------------------------
def prepare_packet_json(paxos_id: str, version: int, bnum: int, bcoord: int, first_undecided_slot: int) -> bytes:
    """PreparePacket.toJSONObjectImpl :78-86 (the same object journal.prepare_json journals)"""
    d = _base(PT_PREPARE, paxos_id, version)
    d.update({"B": f"{int(bnum)}:{int(bcoord)}", "PREP_MIN": int(first_undecided_slot)})
    return _dumps(d)


def _request_obj(paxos_id, version, pt, req_id, value: bytes, entry_replica, entry_time, stop) -> dict:
    """RequestPacket.toJSONObjectImpl :652-695 (the keys this path sets: QID, QV, ET, E, STOP)"""
    d = _base(pt, paxos_id, version)
    d.update({"QID": int(req_id), "QV": bytes(value).decode(CHARSET), "ET": int(entry_time), "E": int(entry_replica)})
    if stop:
        d["STOP"] = True
    return d


def _request_smart(r, pt: int) -> dict:
    d = _base(pt, r.paxos_id, r.version)
    d.update({"QID": int(r.request_id), "QV": bytes(r.value).decode(CHARSET)})
    if r.response:
        d["RV"] = bytes(r.response).decode(CHARSET)
    d["ET"] = int(r.entry_time)
    if r.forward_count > 0:
        d["NFWDS"] = int(r.forward_count)
    if r.stop:
        d["STOP"] = True
    d["E"] = int(r.entry_replica)
    for key, a in (("CA", r.client), ("LA", r.listen)):
        if a is not None:
            d[key] = f"/{a[0]}:{int(a[1])}"  # InetSocketAddress.toString() of a literal address
    if r.should_return:
        d["QF"] = True
    if r.batched:
        d["BATCH"] = [_request_smart(b, PT_REQUEST) for b in r.batched]
    if r.broadcasted:
        d["BC"] = True
    if r.digest:
        d["DIG"] = bytes(r.digest).decode(CHARSET)
    return d


def request_json(r, pt: int = PT_REQUEST) -> bytes:
    """RequestPacket.toJSONSmartImpl :697-742 of a wire.Request: QID, QV, RV (a response), ET, NFWDS (forwardCount > 0),
    STOP, E, CA and LA (InetSocketAddress.toString(): "/1.2.3.4:5678"), QF, BATCH (the batched requests' own objects),
    BC and DIG, over PaxosPacket's type / PT / ID / V.  A Java peer's forwarded requests arrive in this form, as members
    of a batched_paxos_packet_json wrapper."""
    return _dumps(_request_smart(r, pt))


def _org_quote(s: str) -> str:
    """org.json JSONObject.quote: '"', '\\\\' and '/' after '<' escaped, \\b \\t \\n \\f \\r, every other character below
    U+0020, U+0080-U+009F and U+2000-U+20FF as \\uXXXX"""
    out, prev = ['"'], ""
    for c in s:
        if c in '"\\':
            out.append("\\" + c)
        elif c == "/":
            out.append("\\/" if prev == "<" else "/")
        elif c in "\b\t\n\f\r":
            out.append({"\b": "\\b", "\t": "\\t", "\n": "\\n", "\f": "\\f", "\r": "\\r"}[c])
        elif c < " " or "\x80" <= c < "\xa0" or "\u2000" <= c < "\u2100":
            out.append("\\u%04x" % ord(c))
        else:
            out.append(c)
        prev = c
    return "".join(out + ['"'])


def _org_value(v) -> str:
    if isinstance(v, bool):
        return "true" if v else "false"
    if isinstance(v, int):
        return str(v)
    if isinstance(v, str):
        return _org_quote(v)
    if isinstance(v, list):
        return "[" + ",".join(_org_value(x) for x in v) + "]"
    return "{" + ",".join(_org_quote(k) + ":" + _org_value(x) for k, x in v.items()) + "}"


def _request_org(r, pt: int) -> dict:
    """PaxosPacket.toJSONObject :478-494 over RequestPacket.toJSONObjectImpl :652-694, keys in the order they are put"""
    d = _base(pt, r.paxos_id, r.version)
    d.update({"QID": int(r.request_id), "QV": bytes(r.value).decode(CHARSET)})
    if r.response:
        d["RV"] = bytes(r.response).decode(CHARSET)
    d["ET"] = int(r.entry_time)
    if r.forward_count > 0:
        d["NFWDS"] = int(r.forward_count)
    if r.stop:
        d["STOP"] = True
    d["E"] = int(r.entry_replica)
    for key, a in (("CA", r.client), ("LA", r.listen)):
        if a is not None:
            d[key] = f"/{a[0]}:{int(a[1])}"  # the InetSocketAddress, written by its toString()
    if r.should_return:
        d["QF"] = True
    if r.batched:
        d["BATCH"] = [_request_org(b, PT_REQUEST) for b in r.batched]
    if r.broadcasted:
        d["BC"] = True
    if r.digest:
        d["DIG"] = bytes(r.digest).decode(CHARSET)
    return d


def client_request_json(r, sender=None, receiver=None, smart: bool = False) -> bytes:
    """What a gigapaxos client sends for a wire.Request (PaxosClientAsync.sendRequest :165-172: request.toJSONObject()),
    a bare JSON object in org.json's form: keys in toJSONObjectImpl order, strings quoted as JSONObject.quote does,
    ISO-8859-1 bytes.  A client's own request has no clientAddress, so r.client is normally None and there is no "CA".
    smart: the json-smart form instead (request_json's object).
    sender / receiver ((ip, port)): the stamps a receiver adds (MessageExtractor.stampAddressIntoJSONObject :348-376)
    unless the key is present: org.json "_SNDR_ADDRESS":"a.b.c.d:port" (with the deprecated "_SNDR_IP" / "_SNDR_PORT")
    and "_RCVR_ADDRESS", json-smart the InetSocketAddress.toString() form "/a.b.c.d:port"."""
    d = _request_smart(r, PT_REQUEST) if smart else _request_org(r, PT_REQUEST)
    if sender is not None:
        d.setdefault("_SNDR_ADDRESS", f"/{sender[0]}:{int(sender[1])}" if smart else f"{sender[0]}:{int(sender[1])}")
        if not smart:
            d.setdefault("_SNDR_IP", str(sender[0]))
            d.setdefault("_SNDR_PORT", int(sender[1]))
    if receiver is not None:
        d.setdefault("_RCVR_ADDRESS",
                     f"/{receiver[0]}:{int(receiver[1])}" if smart else f"{receiver[0]}:{int(receiver[1])}")
    return _dumps(d) if smart else _org_value(d).encode(CHARSET)


def accepted_pvalue_obj(paxos_id: str, version: int, pv, blob: bytes, entry_replica: int = -1, entry_time: int = 0,
                        pt: int = PT_ACCEPT) -> dict:
    """One entry of ACC_MAP: the PValuePacket JSON (PaxosPacket.toJSONObject :478-494 + PValuePacket.toJSONObjectImpl
    :184-193 {"B", "GC_S"} + ProposalPacket :63-67 {"S"} + the request) of an accepted pvalue record
    (abi.accepted_pvalue_dtype) whose request body is `blob` in the engine's form: the raw requestValue for one request,
    nreq x {reqID, len, flags} + the values for a batched slot (RequestPacket.batched -> "BATCH")."""
    import numpy as np
    from . import abi
    nreq = int(pv["flags"]) >> 16
    stop = bool(int(pv["flags"]) & 2)
    if nreq <= 1:
        d = _request_obj(paxos_id, version, pt, int(pv["req_id"]), blob, entry_replica, entry_time, stop)
    else:
        ents = np.frombuffer(blob[: 16 * nreq], dtype=abi.batch_ent_dtype)
        off, objs = 16 * nreq, []
        for e in ents:
            objs.append(_request_obj(paxos_id, version, PT_REQUEST, int(e["req_id"]), blob[off: off + int(e["len"])],
                                     entry_replica, entry_time, bool(int(e["flags"]) & abi.F_STOP)))
            off += int(e["len"])
        d = dict(objs[0])
        d["PT"] = pt
        d["BATCH"] = objs[1:]  # the first request carries the ones latched along (RequestPacket.latchToBatch); the slot is
        # a stop when any of them is (RequestPacket.isStopRequest: stop || isAnyBatchedRequestStop)
    d.update({"B": f"{int(pv['bnum'])}:{int(pv['bcoord'])}", "GC_S": -1, "S": int(pv["slot"])})
    return d


def prepare_reply_json(paxos_id: str, version: int, acceptor: int, bnum: int, bcoord: int, gc_slot: int,
                       accepted: Sequence[dict], create_time: int = 0) -> bytes:
    """PrepareReplyPacket(receiverID, ballot, accepted, gcSlot) :89-93 -> toJSONObjectImpl :131-143.  firstSlot = gcSlot + 1;
    MIN_S / MAX_S are the static getMinSlot / getMaxSlot :166-190 over the accepted slots (firstSlot when there are none),
    TOT_S their number (all three serve PrepareReplyAssembler's de-fragmentation)."""
    first = _i32(int(gc_slot) + 1)
    lo = hi = None
    for a in accepted:
        s = int(a["S"])
        lo = s if lo is None or _i32(s - lo) < 0 else lo
        hi = s if hi is None or _i32(s - hi) > 0 else hi
    d = _base(PT_PREPARE_REPLY, paxos_id, version)
    d.update({"ACCPTR": int(acceptor), "B": f"{int(bnum)}:{int(bcoord)}", "ACC_MAP": list(accepted), "PREPLY_MIN": first,
              "MAX_S": first if hi is None else hi, "MIN_S": first if lo is None else lo, "TOT_S": len(accepted),
              "CT": int(create_time)})
    return _dumps(d)


def prepare_replies_to_packets(replies, names: Dict[int, Tuple[str, int]], node_of_lane: Sequence[int], read_body) -> List[bytes]:
    """gpx_handle_prepares' reply records (abi.prepare_reply_dtype, reply of PREPARE i at lane l at index i * L + l) as the
    PREPARE_REPLY packets a Java coordinator expects.  read_body(lane, frame_ref, nbytes) -> the request blob from that
    acceptor's log ring (Engine.log_read(lane, frame_ref * 16, nbytes))."""
    from . import abi
    L = len(node_of_lane)
    out = []
    for k, r in enumerate(replies):
        who = int(r["who"])
        if (who >> 16) & abi.F_VOID:
            continue
        lane = k % L
        pid, ver = names[int(r["gid"])]
        acc = [accepted_pvalue_obj(pid, ver, pv, read_body(lane, int(pv["frame_ref"]), int(pv["payload_len"])))
               for pv in r["accepted"][: int(r["n_accepted"])]]
        out.append(prepare_reply_json(pid, ver, node_of_lane[lane], int(r["bnum"]), int(r["bcoord"]), int(r["first_slot"]), acc))
    return out


def _pvalue_blob(a: dict):
    """ACC_MAP entry -> (req_id, blob in the engine's form, nreq, stop)"""
    import numpy as np
    from . import abi
    reqs = [a] + list(a.get("BATCH", []))
    stop = any(bool(q.get("STOP", False)) for q in reqs)
    if len(reqs) == 1:
        return int(a["QID"]), a["QV"].encode(CHARSET), 1, stop
    ents = np.zeros(len(reqs), dtype=abi.batch_ent_dtype)
    vals = []
    for i, q in enumerate(reqs):
        v = q["QV"].encode(CHARSET)
        ents[i]["req_id"], ents[i]["len"] = int(q["QID"]), len(v)
        ents[i]["flags"] = abi.F_STOP if q.get("STOP", False) else 0
        vals.append(v)
    return int(a["QID"]), ents.tobytes() + b"".join(vals), len(reqs), stop


def prepare_reply_to_records(pkt: Packet, gid: int, members: Sequence[int], preparer: int):
    """A PREPARE_REPLY packet from a (remote) acceptor as the input of gpx_handle_prepare_replies: -> (records
    [abi.prepare_reply_dtype], arena bytes).  More than GPX_MAX_WINDOW accepted pvalues continue in further records of
    the same acceptor flagged GPX_F_MORE; the pvalues' frame_ref is the 16-byte unit offset of the request blob in the
    returned arena (the caller adds the position it copies the arena to)."""
    import numpy as np
    from . import abi
    j = pkt if isinstance(pkt, dict) else _loads(pkt)
    assert j["type"] == PT_PAXOS_PACKET and j["PT"] == PT_PREPARE_REPLY
    bn, bc = (int(x) for x in j["B"].split(":"))
    members = list(members)
    idx = members.index(int(j["ACCPTR"])) if int(j["ACCPTR"]) in members else 0xFF
    dst = members.index(int(preparer)) if int(preparer) in members else 0xFF
    acc = sorted(j.get("ACC_MAP", []), key=lambda a: int(a["S"]))  # TreeMap<Integer, PValuePacket>
    arena = bytearray()
    pvs = []
    for a in acc:
        rid, blob, nreq, stop = _pvalue_blob(a)
        abn, abc = (int(x) for x in a["B"].split(":"))
        pv = np.zeros((), dtype=abi.accepted_pvalue_dtype)
        pv["slot"], pv["bnum"], pv["bcoord"], pv["frame_ref"] = int(a["S"]), abn, abc, len(arena) // 16
        pv["req_id"], pv["payload_len"], pv["flags"] = rid, len(blob), (2 if stop else 0) | (nreq << 16)
        arena += blob + bytes(-len(blob) % 16)
        pvs.append(pv)
    chunks = [pvs[k: k + abi.GPX_MAX_WINDOW] for k in range(0, len(pvs), abi.GPX_MAX_WINDOW)] or [[]]
    recs = np.zeros(len(chunks), dtype=abi.prepare_reply_dtype)
    for ci, ch in enumerate(chunks):
        r = recs[ci]
        r["gid"], r["first_slot"], r["bnum"], r["bcoord"] = gid, _i32(int(j["PREPLY_MIN"]) - 1), bn, bc
        r["who"] = abi.who(idx, dst, abi.F_MORE if ci + 1 < len(chunks) else 0)
        r["n_accepted"] = len(ch)
        for k, pv in enumerate(ch):
            r["accepted"][k] = pv
    return recs, bytes(arena)


# ---- SYNC_DECISIONS and the decisions that answer it ----------------------------------------------------------------
def sync_decisions_json(paxos_id: str, version: int, node: int, max_decision_slot: int, missing: Sequence[int]) -> bytes:
    """SyncDecisionsPacket.toJSONObjectImpl :79-88"""
    d = _base(PT_SYNC_DECISIONS, paxos_id, version)
    d.update({"SNDR": int(node), "MAX_S": int(max_decision_slot)})
    if len(missing):
        d["MISS"] = [int(x) for x in missing]
    return _dumps(d)


def serve_sync_request(engine, lane: int, gid: int, pkt: Packet, max_committed_slot: int) -> List[bytes]:
    """PISM.handleSyncDecisionsPacket :2426-2510 at the donor `lane` of `engine`: the logged decisions from the first
    missing slot up to maxDecisionSlot -- or, when the requester knows of none (maxDecisionSlot <= minMissingSlot), up to
    what this replica has committed (:2470-2483) -- each with the request body of the logged accept of its slot
    (getActualDecisions :2539-2583), as DECISION packets.  The journal is looked up by gpx_log_find, the bodies come
    back in one gpx_log_gather."""
    import numpy as np
    from . import abi
    j = pkt if isinstance(pkt, dict) else _loads(pkt)
    assert j["type"] == PT_PAXOS_PACKET and j["PT"] == PT_SYNC_DECISIONS
    missing = [int(x) for x in j.get("MISS", [])]
    if not missing:
        return []
    lo = missing[0]
    hi = int(j["MAX_S"]) if _i32(int(j["MAX_S"]) - lo) > 0 else max(lo + 1, int(max_committed_slot) + 1)
    filt = set(missing) if _i32(int(j["MAX_S"]) - lo) > 0 else None  # :2485-2494: only the slots reported missing
    hits = []
    sl = lo
    while _i32(hi - sl) > 0:
        w = np.zeros(1, dtype=abi.log_want_dtype)
        w["gid"], w["min_slot"], w["n_slots"] = gid, sl, min(abi.GPX_LOG_SPAN, _i32(hi - sl))
        for h in engine.log_find(lane, w)[0][: int(w["n_slots"][0])]:
            d, a = h["decision"], h["accept"]
            if int(d["flags"]) & abi.F_VOID or int(a["flags"]) & abi.F_VOID:
                continue  # "has no body for executed meta-decision" :2570: left out
            if filt is not None and int(d["slot"]) not in filt:
                continue
            hits.append(h.copy())
        sl = _i32(sl + abi.GPX_LOG_SPAN)
    bodies = engine.log_gather(lane, [int(h["blob_pos"]) for h in hits], [int(h["accept"]["payload_len"]) for h in hits])
    out = []
    for h, body in zip(hits, bodies):
        d, a = h["decision"], h["accept"]
        pv = np.zeros((), dtype=abi.accepted_pvalue_dtype)
        pv["slot"], pv["bnum"], pv["bcoord"], pv["req_id"] = int(a["slot"]), int(a["bnum"]), int(a["bcoord"]), int(a["req_id"])
        pv["payload_len"] = int(a["payload_len"])
        pv["flags"] = (2 if int(a["flags"]) & abi.F_STOP else 0) | (int(a["nreq"]) << 16)
        obj = accepted_pvalue_obj(j["ID"], j["V"], pv, body, pt=PT_DECISION)
        obj["GC_S"] = max(int(d["median_cp"]), -1)  # pvalue.makeDecision(getMedianCheckpointedSlot()) :2561
        out.append(_dumps(obj))
    return out


def decisions_to_records(pkts: Sequence[Packet], gid: int, lane: int):
    """DECISION packets with values (a sync reply) -> what replays them at `lane`: (accept records, blob arena, decision
    records), slot order -- the ACCEPT carries the value into the acceptor's window, the DECISION commits it
    (PISM.handleCommittedRequest :1432)."""
    import numpy as np
    from . import abi
    objs = sorted((p if isinstance(p, dict) else _loads(p) for p in pkts), key=lambda o: _i32(int(o["S"])))
    acc = np.zeros(len(objs), dtype=abi.accept_dtype)
    dec = np.zeros(len(objs), dtype=abi.decision_dtype)
    arena = bytearray()
    for k, o in enumerate(objs):
        assert o["PT"] == PT_DECISION
        rid, blob, nreq, stop = _pvalue_blob(o)
        bn, bc = (int(x) for x in o["B"].split(":"))
        for r in (acc[k], dec[k]):
            r["gid"], r["slot"], r["bnum"], r["bcoord"], r["req_id"], r["dst_mask"] = gid, int(o["S"]), bn, bc, rid, 1 << lane
        acc[k]["median_cp"], acc[k]["flags"] = -1, abi.F_ACCEPT | (abi.F_STOP if stop else 0)
        acc[k]["payload_off"], acc[k]["payload_len"], acc[k]["nreq"], acc[k]["sender"] = len(arena), len(blob), nreq, bc
        dec[k]["median_cp"], dec[k]["flags"] = int(o["GC_S"]), abi.F_DECISION | (abi.F_STOP if stop else 0)
        arena += blob + bytes(-len(blob) % 16)
    return acc, np.frombuffer(bytes(arena), dtype=np.uint8), dec


# ---- BATCHED_PAXOS_PACKET ------------------------------------------------------------------------------------------
Packet = Union[bytes, dict]
"""a packet on its way out: byteified (bytes not starting with '{'), a JSON string (bytes starting with '{') or a dict"""


def _as_obj(p: Packet):
    if isinstance(p, dict):
        return p
    if p[:1] == b"{":
        return _loads(p)
    raise ValueError("a BatchedPaxosPacket holds JSON packets: byteified packets are sent on their own "
                     "(BatchedPaxosPacket.toJSONObjectImpl calls toJSONObject on every member)")


def batched_paxos_packet_json(packets: Sequence[Packet]) -> bytes:
    """BatchedPaxosPacket: paxosID null (the key is absent), version -1 (PaxosPacket((PaxosPacket) null) :399-405)"""
    assert len(packets) > 0
    d = _base(PT_BATCHED_PAXOS_PACKET, None, -1)
    d["PP"] = [_as_obj(p) for p in packets]
    return _dumps(d)


def unbatch(packet: bytes) -> List[dict]:
    """PaxosManager.handleIncomingPacket :1087-1090: the member packets of a BATCHED_PAXOS_PACKET (any other JSON packet:
    itself)"""
    j = _loads(packet)
    assert j["type"] == PT_PAXOS_PACKET
    return list(j["PP"]) if j["PT"] == PT_BATCHED_PAXOS_PACKET else [j]


MessagingTask = Tuple[Sequence[int], Sequence[Packet]]
"""(recipients, msgs) -- paxosutil/MessagingTask"""


def batch_messaging_tasks(tasks: Sequence[MessagingTask], batch_across_groups: bool = BATCH_ACROSS_GROUPS,
                          min_pp_batch_size: int = MIN_PP_BATCH_SIZE) -> List[Tuple[List[int], List[bytes]]]:
    """PaxosPacketBatcher.process :270-277 + batch :280-303.  Returns (recipients, [wire messages]) per send.  Byteified
    members of a group of tasks cannot ride in the JSON wrapper; they are sent beside it, as the messenger does for a
    MessagingTask whose packets are Byteable (PaxosMessenger.toObjects :156-166)."""
    live = [(list(r), list(m)) for r, m in tasks if r is not None and len(r) and m is not None and len(m)]
    if not (batch_across_groups and len(tasks) > min_pp_batch_size):
        return [(r, [p if isinstance(p, bytes) else _dumps(p) for p in m]) for r, m in live]
    grouped: Dict[frozenset, List[Packet]] = {}
    for r, m in live:  # dict preserves first-seen order like the LinkedHashMap
        grouped.setdefault(frozenset(int(x) for x in r), []).extend(m)
    out = []
    for group, msgs in grouped.items():
        js = [p for p in msgs if isinstance(p, dict) or p[:1] == b"{"]
        raw = [p for p in msgs if not (isinstance(p, dict) or p[:1] == b"{")]
        wire = list(raw)
        if js:
            wire.append(batched_paxos_packet_json(js))
        out.append((sorted(group), wire))
    return out


def parse_packet(pkt: bytes) -> dict:
    """journal.parse_packet extended by the types above: {"kind": ...}"""
    from . import journal
    if pkt[:1] != b"{":
        return journal.parse_packet(pkt)
    j = _loads(pkt)
    pt = j["PT"]
    if pt == PT_ACCEPT_REPLY:
        bn, bc = (int(x) for x in j["B"].split(":"))
        return {"kind": "ACCEPT_REPLY", "paxos_id": j["ID"], "version": j["V"], "acceptor": j["SNDR"], "bnum": bn,
                "bcoord": bc, "slot_number": j["S"], "max_checkpointed_slot": j["CP_S"], "request_id": j["QID"],
                "undigest_request": bool(j.get("NACK", False))}
    if pt == PT_BATCHED_ACCEPT_REPLY:  # BatchedAcceptReply(JSONObject) :64-72
        bn, bc = (int(x) for x in j["B"].split(":"))
        pairs = [int(x) for x in j["SLOTS"]]
        if len(pairs) % 2:
            raise ValueError("SLOTS of odd length")
        return {"kind": "BATCHED_ACCEPT_REPLY", "paxos_id": j["ID"], "version": j["V"], "acceptor": j["SNDR"],
                "bnum": bn, "bcoord": bc, "slot_number": j["S"], "max_checkpointed_slot": j["CP_S"],
                "request_id": j["QID"], "slots": pairs[0::2], "request_ids": pairs[1::2]}
    if pt == PT_BATCHED_COMMIT:  # BatchedCommit(JSONObject) :75-92
        bn, bc = (int(x) for x in j["B"].split(":"))
        return {"kind": "BATCHED_COMMIT", "paxos_id": j["ID"], "version": j["V"], "bnum": bn, "bcoord": bc,
                "median_cp": j["GC_S"], "group": [int(x) for x in j["GROUP"]], "slots": [int(x) for x in j["SLOTS"]]}
    if pt == PT_BATCHED_ACCEPT:
        b = BatchedAccept.from_json(j)
        return {"kind": "BATCHED_ACCEPT", "paxos_id": b.paxos_id, "version": b.version, "bnum": b.bnum, "bcoord": b.bcoord,
                "median_cp": b.median_cp, "group": b.group, "slot_digests": dict(b.slot_digests),
                "slot_request_ids": dict(b.slot_request_ids)}
    if pt == PT_SYNC_DECISIONS:
        return {"kind": "SYNC_DECISIONS", "paxos_id": j["ID"], "version": j["V"], "node": j["SNDR"],
                "max_decision_slot": j["MAX_S"], "missing": [int(x) for x in j.get("MISS", [])]}
    if pt == PT_PREPARE_REPLY:
        bn, bc = (int(x) for x in j["B"].split(":"))
        return {"kind": "PREPARE_REPLY", "paxos_id": j["ID"], "version": j["V"], "acceptor": j["ACCPTR"], "bnum": bn,
                "bcoord": bc, "first_slot": j["PREPLY_MIN"], "min_slot": j["MIN_S"], "max_slot": j["MAX_S"],
                "total_count": j["TOT_S"], "accepted_slots": sorted(int(a["S"]) for a in j.get("ACC_MAP", []))}
    if pt == PT_BATCHED_PAXOS_PACKET:
        return {"kind": "BATCHED_PAXOS_PACKET", "packets": [parse_packet(_dumps(p)) for p in j["PP"]]}
    return journal.parse_packet(pkt)
