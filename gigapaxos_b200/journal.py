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
from .paxos_manager import _jsub

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

    def append_frames(self, frames):
        """frames already in the {int32 BE len}{bytes} form (gpx_log_frame_device's output), in one write"""
        self.fos.write(frames)
        self.cur_size += len(frames)

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


MetaSource = Callable[[np.ndarray], np.ndarray]
"""journal_miss_dtype records -> journal_req_dtype records: {gid, entryReplica, req_id, entryTime} of the requests a
frame call lacks (PaxosManager.outstanding is the Java node's source)."""


class DeviceLogDrainer:
    """LogDrainer's job with the frames written on the device (gpx_log_frame_device): one call frames every image of
    the lane's undrained range in HBM, the frames come down to page-locked memory in one copy and go to the Journaler in
    one write, then the range is released.  The caller's table of entryReplica / entryTime lives on the device; add()
    puts requests in it ahead of the drain, and the requests a call reports missing (GPX_ENOENT) are asked of
    meta_source before the call is repeated."""

    def __init__(self, engine: Engine, lane: int, journaler: Journaler, meta_source: MetaSource, offset: int = 0):
        self.engine, self.lane, self.j, self.meta_source = engine, lane, journaler, meta_source
        self.offset = offset
        self.frames_written = 0
        self.meta = np.zeros(0, dtype=abi.journal_req_dtype)
        self._dmeta = None
        self._pinned = None
        self.caps = (1 << 16, 1 << 10, 64)

    def add(self, reqs: np.ndarray):
        """enter journal_req_dtype records in the table (a request already in it keeps its entry)"""
        reqs = np.asarray(reqs, dtype=abi.journal_req_dtype)
        if len(reqs) == 0:
            return
        m = np.concatenate([self.meta, reqs])
        m = m[np.lexsort((m["req_id"], m["gid"]))]  # stable: of equal keys the table's entry comes first
        new = np.ones(len(m), dtype=bool)
        new[1:] = (m["gid"][1:] != m["gid"][:-1]) | (m["req_id"][1:] != m["req_id"][:-1])
        self.meta = m[new]
        self._dmeta = None

    def forget(self, keep: np.ndarray):
        """keep only the table entries where keep (a bool mask over self.meta) is true"""
        self.meta = self.meta[keep]
        self._dmeta = None

    def _device_meta(self):
        import torch
        if self._dmeta is None and len(self.meta):
            self._dmeta = torch.from_numpy(self.meta.view(np.uint8).reshape(-1, 24).copy()).cuda()
        return self._dmeta

    def drain(self) -> int:
        """frames [offset, head) into the journal; returns the number of frames"""
        import torch
        while True:
            r = self.engine.log_frame_device(self.lane, self.offset, self._device_meta(), len(self.meta), self.caps)
            self.caps = tuple(max(a, b) for a, b in zip(self.caps, r.sizes))
            if r.rc == abi.GPX_OK:
                break
            torch.cuda.current_stream().synchronize()
            miss = np.ascontiguousarray(r.missing.cpu().numpy()).reshape(-1).view(abi.journal_miss_dtype)
            if np.any(miss["req_id"] == -1):
                raise KeyError("gids without a name (gpx_set_group_names): %s" % sorted(set(miss["gid"].tolist())))
            before = len(self.meta)
            self.add(self.meta_source(miss))
            if len(self.meta) == before:
                raise KeyError("meta_source knows none of %d missing requests" % len(miss))
        n = int(r.sizes[0])
        if n:
            if self._pinned is None or self._pinned.numel() < n:
                self._pinned = torch.empty(max(n, 1 << 20), dtype=torch.uint8, pin_memory=True)
            self._pinned[:n].copy_(r.frames[:n], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            self.j.append_frames(memoryview(self._pinned[:n].numpy()))
        self.j.end_batch()
        self.frames_written += int(r.sizes[1])
        self.offset = r.from_
        self.engine.log_release(self.lane, self.offset)
        return int(r.sizes[1])


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


# ---- garbage collection (SQLPaxosLogger.garbageCollectJournal :3154, compactLogfiles :3282-3450, mergeLogfiles :3476)

JGC_UNCHANGED, JGC_COMPACTED, JGC_EMPTY, JGC_TORN = 0, 1, 2, 3  # gpx_journal_file.status


GcSlotOf = Callable[[str, int], "int | None"]
"""(paxosID, version) -> the group's GC slot, or None when the pair names no live group (gpx_set_group_names' table)."""


class CompactedFile:
    """what compaction does to one journal file: status (JGC_*), the new bytes of a JGC_COMPACTED file, the frames it
    holds afterwards and those removed, and how many of its frames named no live group"""

    def __init__(self, status: int, data, kept: int, dropped: int, unresolved: int):
        self.status, self.data, self.kept, self.dropped, self.unresolved = status, data, kept, dropped, unresolved

    def __eq__(self, other):
        return vars(self) == vars(other)

    def __repr__(self):
        return "CompactedFile(%r)" % {k: (len(v) if k == "data" and v is not None else v) for k, v in vars(self).items()}


def _frames(data: bytes):
    """(offset, packet) of every whole frame, and where read_journal's walk stops"""
    out, p = [], 0
    while p + 4 <= len(data):
        (ln,) = struct.unpack(">i", data[p: p + 4])
        if ln < 0 or p + 4 + ln > len(data):
            break
        out.append((p, data[p + 4: p + 4 + ln]))
        p += 4 + ln
    return out, p


def _gc_fields(pkt: bytes):
    """(paxosID, version, slot, bnum, bcoord, is_prepare) of a journaled packet, or ValueError"""
    try:
        v = parse_packet(pkt)
    except Exception as e:  # noqa: BLE001 -- any failure to read the packet is a malformed frame
        raise ValueError("frame does not parse: %s" % e) from None
    slot = v["first_undecided_slot"] if v["kind"] == "PREPARE" else v["slot"]
    ints = [v["version"], slot, v["bnum"], v["bcoord"]]
    if not isinstance(v["paxos_id"], str) or any(type(x) is not int or not -(1 << 31) <= x < (1 << 31) for x in ints):
        raise ValueError("frame fields out of range")
    return v["paxos_id"], v["version"], slot, v["bnum"], v["bcoord"], v["kind"] == "PREPARE"


def compact_files(files: List[str], gc_slot_of: GcSlotOf, last_readonly: bool = True) -> List[CompactedFile]:
    """The host model of gpx_journal_compact_device (include/gpx.h): one lane's journal files in roll order -> what
    compaction does to each.  A frame whose (paxosID, version) names no live group is kept; one at or below its
    group's GC slot is dropped; a PREPARE is also dropped when an indexed frame of its group (any frame above the GC
    slot, in any of the files) has a higher ballot, compared entry by entry as LogIndex.isLogMsgNeeded :331-345 does.
    An ACCEPT's or DECISION's slot is its pvalue's slot (the index's, MessageLogDiskMap.add :412), not the ballot
    number SQLPaxosLogger.getSlot :492-496 returns.  A torn file, and the last one when last_readonly, stay as they
    are.  ValueError on a frame that is not an ACCEPT, a DECISION or a PREPARE."""
    parsed = []  # per file: (data, [(offset, length, group key or None, indexed, fields)], torn)
    index: Dict[tuple, List[Tuple[int, int]]] = {}
    for path in files:
        with open(path, "rb") as f:
            data = f.read()
        frames, end = _frames(data)
        rows = []
        for k, (off, pkt) in enumerate(frames):
            try:
                pid, ver, slot, bn, bc, prep = _gc_fields(pkt)
            except ValueError as e:
                raise ValueError("%s: frame %d: %s" % (path, k, e)) from None
            gc = gc_slot_of(pid, ver)
            key = None if gc is None else (pid, ver)
            indexed = key is not None and _jsub(slot, gc) > 0
            if indexed:
                index.setdefault(key, []).append((bn, bc))
            rows.append((off, 4 + len(pkt), key, indexed, prep, bn, bc))
        parsed.append((data, rows, end != len(data)))
    out = []
    for i, (data, rows, torn) in enumerate(parsed):
        keep = []
        for off, ln, key, indexed, prep, bn, bc in rows:
            if key is None:
                k = True
            elif not indexed:
                k = False
            elif prep:
                k = not any(_jsub(en, bn) > 0 or (en == bn and _jsub(ec, bc) > 0) for en, ec in index[key])
            else:
                k = True
            keep.append(k)
        unresolved = sum(1 for r in rows if r[2] is None)
        kept = sum(keep)
        if torn or (last_readonly and i == len(parsed) - 1):
            out.append(CompactedFile(JGC_TORN if torn else JGC_UNCHANGED, None, len(rows), 0, unresolved))
        elif kept == 0:
            out.append(CompactedFile(JGC_EMPTY, None, 0, len(rows), unresolved))
        elif kept == len(rows):
            out.append(CompactedFile(JGC_UNCHANGED, None, kept, 0, unresolved))
        else:
            body = b"".join(data[off: off + ln] for (off, ln, *_), k in zip(rows, keep) if k)
            out.append(CompactedFile(JGC_COMPACTED, body, kept, len(rows) - kept, unresolved))
    return out


def _replace(path: str, data) -> None:
    """path's contents become data: a .tmp file written, fsynced and renamed over it (modifyLogfileAndLogIndex)"""
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        f.write(data)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


def apply_compaction(journaler: Journaler, files: List[str], results: List[CompactedFile]) -> None:
    """Writes what compaction decided for each of files (journaler's, the current file never among them): a
    compacted file replaced, an empty one deleted and dropped from journaler.files.  Then adjacent files whose sizes
    sum to at most 2 x the journaler's file size limit are merged into the later one, the earlier deleted
    (compactLogfiles :3305-3312 / mergeLogfiles).  A torn file is neither merged nor merged into: its tail would end
    up inside the merged file."""
    if journaler.cur in files:
        raise ValueError("the current journal file is never rewritten")
    left = []
    for path, r in zip(files, results):
        if r.status == JGC_COMPACTED:
            _replace(path, r.data)
        elif r.status == JGC_EMPTY:
            os.remove(path)
            journaler.files.remove(path)
            continue
        left.append((path, r.status == JGC_TORN))
    prev = None
    for path, torn in left:
        if torn:
            prev = None
            continue
        if prev is not None and os.path.getsize(prev) + os.path.getsize(path) <= 2 * journaler.max:
            with open(prev, "rb") as a, open(path, "rb") as b:
                _replace(path, a.read() + b.read())
            os.remove(prev)
            journaler.files.remove(prev)
        prev = path


class JournalCompactor:
    """Garbage-collects a Journaler's files on the device (gpx_journal_compact_device): the files but the current one
    are read, indexed on the host (gpx_journal_index), uploaded once together with the current file (read-only: its
    frames still count for the PREPARE rule), compacted in one call, and written back by apply_compaction."""

    def __init__(self, engine: Engine, journaler: Journaler):
        self.engine, self.j = engine, journaler
        self.caps = (1 << 20, 64)

    def compact(self, gc_slot: np.ndarray) -> List[CompactedFile]:
        """gc_slot: int32 per gid of the engine (PaxosManager.journal_gc_slots) -> what happened to each non-current
        file, in the order of journaler.files before the call"""
        import torch
        files = [f for f in self.j.files if f != self.j.cur]
        if not files:
            return []
        self.j.fos.flush()
        blobs = []
        for path in files + [self.j.cur]:
            with open(path, "rb") as f:
                blobs.append(f.read())
        file_off = np.zeros(len(blobs) + 1, np.uint32)
        file_off[1:] = np.cumsum([len(b) for b in blobs])
        starts = np.concatenate([self.engine.L.journal_index(b, int(o)) for b, o in zip(blobs, file_off[:-1])])
        dev = torch.device("cuda", torch.cuda.current_device())
        data = torch.from_numpy(np.frombuffer(b"".join(blobs) or b"\0", np.uint8).copy()).to(dev)
        gcs = torch.from_numpy(np.ascontiguousarray(gc_slot, np.int32)).to(dev)
        r = self.engine.journal_compact_device(data, int(file_off[-1]), torch.from_numpy(file_off).to(dev),
                                               torch.from_numpy(starts.astype(np.uint32)).to(dev), gcs, True,
                                               self.caps)
        self.caps = tuple(max(a, b) for a, b in zip(self.caps, r.sizes))
        if r.rc != abi.GPX_OK:
            raise ValueError("journal frames that do not parse: %s" % r.bad.cpu().numpy().tolist())
        out = r.out.cpu().numpy()
        fr = r.files.cpu().numpy().reshape(-1).view(abi.journal_file_dtype)[: len(files)]
        results = [CompactedFile(int(x["status"]),
                                 out[int(x["out_off"]): int(x["out_off"]) + int(x["out_bytes"])].tobytes()
                                 if int(x["status"]) == JGC_COMPACTED else None,
                                 int(x["kept"]), int(x["dropped"]), int(x["unresolved"])) for x in fr]
        apply_compaction(self.j, files, results)
        return results
