"""Journal persistence: drain the engine's HBM log rings into files byte-compatible with the
reference's journal, and read them back (SURVEY.md 8f rank 1).

Mirrors SQLPaxosLogger.Journaler (gigapaxos/SQLPaxosLogger.java:685-848): files
`<logdir>paxos_journal.<node>/log.<node>.<hex millis>`, contents `{int32 BE length}{packet
bytes}*` (journal() :1000-1003, appendToLogFile :814-826), a new file once the current one
exceeds MAX_LOG_FILE_SIZE (rollLogFile :789-812, checked after a batch as in journal() :1041).

What a frame holds is what SQLPaxosLogger.toBytes :1084-1096 produces: ACCEPT packets in the reference's byte codec
(AcceptPacket.toBytes -- BYTEIFICATION), every other packet as the JSON string of PaxosPacket.toString() :1095-1098.
So DECISIONs are journaled as the JSON of the (meta) decision -- PaxosPacket.toJSONObject :478-494 {"type": 90, "PT": 6,
"ID", "V"} + PValuePacket.toJSONObjectImpl :184-193 {"B": "bnum:coord", "GC_S"} + ProposalPacket :63-67 {"S"} +
RequestPacket.toJSONObjectImpl :652-692 {"QID", "ET", "E", "STOP"}; PValuePacket.getMetaDecision :212-218 drops the
request value and sets GC_S = -1 -- and logged PREPAREs as {"type": 90, "PT": 2, "ID", "V", "B", "PREP_MIN"}
(PreparePacket.toJSONObjectImpl :78-86).  A Java SQLPaxosLogger reading these files gets exactly the packet types it
wrote itself; key order inside a JSON object is not significant (org.json).
"""
from __future__ import annotations

import json
import os
import struct
import time
from typing import Callable, Dict, Iterator, List, Tuple

import numpy as np

from . import abi, wire
from .abi import Engine

MAX_LOG_FILE_SIZE = 64 * 1024 * 1024  # PC.MAX_LOG_FILE_SIZE PaxosConfig.java:314


class Journaler:
    """SQLPaxosLogger.Journaler: append-only length-prefixed frames, rolled by size."""

    SUBDIR, PREFIX, POSTPREFIX = "paxos_journal.", "log.", "."

    def __init__(self, logdir: str, node_id, max_log_file_size: int = MAX_LOG_FILE_SIZE):
        self.node_id = node_id
        self.dir = os.path.join(logdir, f"{self.SUBDIR}{node_id}")
        os.makedirs(self.dir, exist_ok=True)
        self.max = max_log_file_size
        self.files: List[str] = []
        self._seq = 0
        self.fos = None
        self.cur_size = 0
        self._create()

    def _name(self) -> str:  # generateLogfileName :729-734 (USE_HEX_TIMESTAMP)
        ts = int(time.time() * 1000) + self._seq
        self._seq += 1
        return os.path.join(self.dir, f"{self.PREFIX}{self.node_id}{self.POSTPREFIX}{ts:x}")

    def _create(self):
        if self.fos:
            self.fos.flush()
            self.fos.close()
        self.cur = self._name()
        self.fos = open(self.cur, "wb")
        self.files.append(self.cur)
        self.cur_size = 0

    def append(self, packet: bytes):
        frame = wire.journal_frame(packet)  # {int32 BE len}{bytes}
        self.fos.write(frame)
        self.cur_size += len(frame)

    def end_batch(self):
        self.fos.flush()  # FLUSH=true, SYNC=false (PaxosConfig.java:720,725)
        if self.cur_size > self.max:
            self._create()

    def close(self):
        if self.fos:
            self.fos.flush()
            self.fos.close()
            self.fos = None


PT_PREPARE, PT_ACCEPT, PT_DECISION, PT_PAXOS_PACKET = 2, 3, 6, 90  # PaxosPacket.PaxosPacketType :206-287


def decision_json(paxos_id: str, version: int, slot: int, bnum: int, bcoord: int, median_cp: int, request_id: int,
                  entry_replica: int, entry_time: int, stop: bool = False) -> bytes:
    """PaxosPacket.toString() of a (meta) DECISION: what SQLPaxosLogger.toString :1095-1098 journals"""
    d = {"type": PT_PAXOS_PACKET, "PT": PT_DECISION, "ID": paxos_id, "V": int(version), "B": f"{int(bnum)}:{int(bcoord)}",
         "GC_S": int(median_cp), "S": int(slot), "QID": int(request_id), "ET": int(entry_time), "E": int(entry_replica)}
    if stop:
        d["STOP"] = True
    return json.dumps(d, separators=(",", ":")).encode("ascii")  # non-ASCII as \uXXXX escapes: charset-neutral


def prepare_json(paxos_id: str, version: int, bnum: int, bcoord: int, first_undecided_slot: int) -> bytes:
    d = {"type": PT_PAXOS_PACKET, "PT": PT_PREPARE, "ID": paxos_id, "V": int(version), "B": f"{int(bnum)}:{int(bcoord)}",
         "PREP_MIN": int(first_undecided_slot)}
    return json.dumps(d, separators=(",", ":")).encode("ascii")  # non-ASCII as \uXXXX escapes: charset-neutral


def parse_packet(pkt: bytes) -> dict:
    """One journaled packet, the way the reference's reader tells them apart (SQLPaxosLogger: a byteified packet starts
    with the int PAXOS_PACKET type, a stringified one with '{'): {"kind": "ACCEPT" | "DECISION" | "PREPARE", ...}"""
    if pkt[:1] == b"{":
        j = json.loads(pkt.decode("iso-8859-1"))  # SQLPaxosLogger.CHARSET :1313 (a Java-written frame may hold raw bytes)
        assert j["type"] == PT_PAXOS_PACKET
        bn, bc = (int(x) for x in j["B"].split(":"))
        if j["PT"] == PT_DECISION:
            return {"kind": "DECISION", "paxos_id": j["ID"], "version": j["V"], "slot": j["S"], "bnum": bn, "bcoord": bc,
                    "median_cp": j["GC_S"], "request_id": j["QID"], "stop": bool(j.get("STOP", False)),
                    "entry_replica": j["E"], "entry_time": j["ET"]}
        if j["PT"] == PT_PREPARE:
            return {"kind": "PREPARE", "paxos_id": j["ID"], "version": j["V"], "bnum": bn, "bcoord": bc,
                    "first_undecided_slot": j["PREP_MIN"]}
        raise ValueError("unexpected packet type %r" % j["PT"])
    v = wire.decode_accept(pkt)
    v["kind"] = "ACCEPT"
    return v


RequestLookup = Callable[[int, int], Tuple[str, int, int, float]]
"""(gid, req_id) -> (paxosID, version, entryReplica, entryTime): the RequestPacket fields the engine
does not carry (PaxosManager keeps them in its outstanding table)."""


class LogDrainer:
    """Drains one lane's log ring into a Journaler, incrementally (the BatchedLogger's role,
    AbstractPaxosLogger.java:691-716, with the device having done the append already)."""

    def __init__(self, engine: Engine, lane: int, journaler: Journaler, lookup: RequestLookup):
        self.engine, self.lane, self.j, self.lookup = engine, lane, journaler, lookup
        self.offset = 0
        self.accepts_written = 0
        self.decisions_written = 0

    def drain(self) -> int:
        head = self.engine.log_head(self.lane)
        if head <= self.offset:
            return 0
        buf = self.engine.log_read(self.lane, self.offset, head - self.offset)
        n = 0
        for hdr, imgs, payload, _ in abi.parse_log(buf, self.engine.cfg.log_ring_bytes, self.offset):
            if int(hdr["rec_bytes"]) == 48:
                for a in imgs:
                    if a["flags"] & abi.F_VOID:
                        continue
                    self.j.append(self._accept_bytes(a, payload))
                    n += 1
                    self.accepts_written += 1
            else:  # DECISION images and logged PREPAREs (GPX_F_PREPARE: the promised ballot) share the 32-byte form
                for dimg in imgs:
                    fl = int(dimg["flags"])
                    if fl & abi.F_VOID:
                        continue
                    try:
                        pid, ver, entry, etime = self.lookup(int(dimg["gid"]), int(dimg["req_id"]))
                    except KeyError:  # a PREPARE carries no request: only (paxosID, version) are needed
                        pid, ver, entry, etime = self.lookup(int(dimg["gid"]), -1)
                    if fl & abi.F_PREPARE:  # the image's slot field carries firstUndecidedSlot
                        self.j.append(prepare_json(pid, ver, int(dimg["bnum"]), int(dimg["bcoord"]), int(dimg["slot"])))
                    else:
                        self.j.append(decision_json(pid, ver, int(dimg["slot"]), int(dimg["bnum"]), int(dimg["bcoord"]),
                                                    int(dimg["median_cp"]), int(dimg["req_id"]), entry, int(etime),
                                                    stop=bool(fl & abi.F_STOP)))
                    self.decisions_written += 1
        self.j.end_batch()
        self.offset = head
        return n

    def _accept_bytes(self, a, payload: np.ndarray) -> bytes:
        off, ln, nreq = int(a["payload_off"]), int(a["payload_len"]), int(a["nreq"])
        blob = payload[off: off + ln].tobytes()
        pid, ver, entry, etime = self.lookup(int(a["gid"]), int(a["req_id"]))
        if nreq <= 1:
            req = wire.Request(pid, ver, int(a["req_id"]), blob, stop=bool(a["flags"] & abi.F_STOP),
                               entry_replica=entry, entry_time=int(etime))
        else:  # RequestPacket.batched: [nreq x {req_id,len,flags}][values]
            ents = np.frombuffer(blob[: 16 * nreq], dtype=abi.batch_ent_dtype)
            vals, p = [], 16 * nreq
            for e in ents:
                vals.append(blob[p: p + int(e["len"])])
                p += int(e["len"])
            subs = []
            for e, v in zip(ents[1:], vals[1:]):
                spid, sver, sentry, setime = self.lookup(int(a["gid"]), int(e["req_id"]))
                subs.append(wire.Request(spid, sver, int(e["req_id"]), v, stop=bool(int(e["flags"]) & abi.F_STOP),
                                         entry_replica=sentry, entry_time=int(setime)))
            req = wire.Request(pid, ver, int(ents[0]["req_id"]), vals[0], stop=bool(int(ents[0]["flags"]) & abi.F_STOP),
                               entry_replica=entry, entry_time=int(etime), batched=tuple(subs))
        return wire.encode_accept(req, int(a["slot"]), int(a["bnum"]), int(a["bcoord"]), False, int(a["median_cp"]),
                                  int(a["sender"]))


def read_journal(path: str) -> Iterator[bytes]:
    """The packets of one journal file (the reader side of {int32 BE len}{bytes}*)."""
    with open(path, "rb") as f:
        data = f.read()
    p = 0
    while p + 4 <= len(data):
        (ln,) = struct.unpack(">i", data[p: p + 4])
        if ln < 0 or p + 4 + ln > len(data):
            break  # torn tail: the reference tolerates a partially written last frame
        yield data[p + 4: p + 4 + ln]
        p += 4 + ln


def replay_accepts(files: List[str]) -> Dict[str, Dict[int, dict]]:
    """Recovery read path (the ACCEPT half of PaxosManager's roll forward, PaxosManager.java:1852-2055):
    per paxosID, the highest-ballot logged ACCEPT of every slot."""
    out: Dict[str, Dict[int, dict]] = {}
    for path in files:
        for pkt in read_journal(path):
            v = parse_packet(pkt)
            if v["kind"] != "ACCEPT":
                continue
            cur = out.setdefault(v["paxos_id"], {}).get(v["slot"])
            if cur is None or (v["bnum"], v["bcoord"]) >= (cur["bnum"], cur["bcoord"]):
                out[v["paxos_id"]][v["slot"]] = v
    return out


def replay_decisions(files: List[str]) -> Dict[str, Dict[int, dict]]:
    """the DECISION half: per paxosID, slot -> the journaled (meta) decision"""
    out: Dict[str, Dict[int, dict]] = {}
    for path in files:
        for pkt in read_journal(path):
            v = parse_packet(pkt)
            if v["kind"] == "DECISION":
                out.setdefault(v["paxos_id"], {})[v["slot"]] = v
    return out
