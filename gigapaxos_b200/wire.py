"""ctypes bindings of include/gpx_wire.h: the reference's big-endian wire / journal byte codecs
(paxospackets/RequestPacket.java:819-1024, AcceptPacket.java:95-138, BatchedAcceptReply.java:103-173,
BatchedCommit.java:184-252, SQLPaxosLogger.java:1000-1003)."""
from __future__ import annotations

import ctypes as C
from collections import namedtuple
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import abi, load_library

PT_REQUEST, PT_ACCEPT, PT_BATCHED_ACCEPT_REPLY, PT_BATCHED_COMMIT = 1, 3, 34, 35


class WireRequest(C.Structure):
    pass


WireRequest._fields_ = [
    ("paxos_id", C.c_char_p), ("paxos_id_len", C.c_uint32), ("version", C.c_int32), ("request_id", C.c_int64),
    ("stop", C.c_uint8), ("client_ip", C.c_uint8 * 4), ("client_port", C.c_uint16), ("listen_ip", C.c_uint8 * 4),
    ("listen_port", C.c_uint16), ("entry_replica", C.c_int32), ("entry_time", C.c_int64),
    ("should_return_request_value", C.c_uint8), ("forward_count", C.c_int32), ("broadcasted", C.c_uint8),
    ("digest", C.c_char_p), ("digest_len", C.c_uint32), ("value", C.c_char_p), ("value_len", C.c_uint32),
    ("response", C.c_char_p), ("response_len", C.c_uint32), ("n_batched", C.c_uint32),
    ("batched", C.POINTER(WireRequest)),
]


class AcceptView(C.Structure):
    _fields_ = [("packet_type", C.c_int32), ("version", C.c_int32), ("paxos_id", C.c_void_p),
                ("paxos_id_len", C.c_uint32), ("request_id", C.c_int64), ("stop", C.c_uint8),
                ("entry_replica", C.c_int32), ("entry_time", C.c_int64), ("value", C.c_void_p),
                ("value_len", C.c_uint32), ("n_batched", C.c_uint32), ("request_bytes", C.c_size_t),
                ("slot", C.c_int32), ("bnum", C.c_int32), ("bcoord", C.c_int32), ("median_cp", C.c_int32),
                ("sender", C.c_int32), ("recovery", C.c_uint8)]


@dataclass
class Request:
    """RequestPacket fields (paxospackets/RequestPacket.java:55-)."""
    paxos_id: str
    version: int
    request_id: int
    value: bytes
    stop: bool = False
    entry_replica: int = -1
    entry_time: int = 0
    client: Optional[tuple] = None  # (ip, port)
    listen: Optional[tuple] = None
    should_return: bool = False
    forward_count: int = 0
    broadcasted: bool = False
    digest: Optional[bytes] = None
    response: bytes = b""
    batched: Sequence["Request"] = field(default_factory=tuple)

    def _c(self, keep: list) -> WireRequest:
        w = WireRequest()
        pid = self.paxos_id.encode("iso-8859-1")
        keep.append(pid)
        w.paxos_id, w.paxos_id_len, w.version, w.request_id = pid, len(pid), self.version, self.request_id
        w.stop = 1 if self.stop else 0
        for name, a in (("client", self.client), ("listen", self.listen)):
            if a is not None:
                ip = [int(x) for x in a[0].split(".")]
                for i in range(4):
                    getattr(w, name + "_ip")[i] = ip[i]
                setattr(w, name + "_port", a[1])
        w.entry_replica, w.entry_time = self.entry_replica, self.entry_time
        w.should_return_request_value = 1 if self.should_return else 0
        w.forward_count, w.broadcasted = self.forward_count, 1 if self.broadcasted else 0
        if self.digest:
            keep.append(self.digest)
            w.digest, w.digest_len = self.digest, len(self.digest)
        keep.append(self.value)
        w.value, w.value_len = self.value, len(self.value)
        keep.append(self.response)
        w.response, w.response_len = self.response, len(self.response)
        if self.batched:
            arr = (WireRequest * len(self.batched))(*[b._c(keep) for b in self.batched])
            keep.append(arr)
            w.n_batched, w.batched = len(self.batched), C.cast(arr, C.POINTER(WireRequest))
        return w


def _lib():
    L = load_library().lib
    L.gpx_wire_encode_request.restype = C.c_size_t
    L.gpx_wire_encode_accept.restype = C.c_size_t
    L.gpx_wire_request_size.restype = C.c_size_t
    L.gpx_wire_encode_batched_accept_reply.restype = C.c_size_t
    L.gpx_wire_encode_batched_commit.restype = C.c_size_t
    L.gpx_wire_journal_frame.restype = C.c_size_t
    return L


def encode_request(r: Request, packet_type: int = PT_REQUEST) -> bytes:
    L, keep = _lib(), []
    w = r._c(keep)
    n = L.gpx_wire_request_size(C.byref(w))
    buf = C.create_string_buffer(n)
    got = L.gpx_wire_encode_request(C.byref(w), C.c_int32(packet_type), buf, C.c_size_t(n))
    assert got == n
    return buf.raw


def encode_accept(r: Request, slot, bnum, bcoord, recovery, median_cp, sender) -> bytes:
    L, keep = _lib(), []
    w = r._c(keep)
    n = L.gpx_wire_request_size(C.byref(w)) + 22
    buf = C.create_string_buffer(n)
    got = L.gpx_wire_encode_accept(C.byref(w), C.c_int32(slot), C.c_int32(bnum), C.c_int32(bcoord),
                                   C.c_uint8(1 if recovery else 0), C.c_int32(median_cp), C.c_int32(sender), buf,
                                   C.c_size_t(n))
    assert got == n
    return buf.raw


def decode_accept(b: bytes) -> dict:
    L = _lib()
    v = AcceptView()
    rc = L.gpx_wire_decode_accept(b, C.c_size_t(len(b)), C.byref(v))
    if rc != 0:
        raise ValueError("malformed ACCEPT")
    out = {k: getattr(v, k) for k in ("packet_type", "version", "request_id", "stop", "entry_replica", "entry_time",
                                      "value_len", "n_batched", "request_bytes", "slot", "bnum", "bcoord",
                                      "median_cp", "sender", "recovery")}
    out["paxos_id"] = b[13: 13 + v.paxos_id_len].decode("iso-8859-1")
    # requestValue: after the header and the 39 fixed bytes comes {int digestLen, digest}{int valueLen, value}
    off = 13 + v.paxos_id_len + 39
    dl = int.from_bytes(b[off: off + 4], "big")
    off += 4 + dl
    out["value"] = b[off + 4: off + 4 + v.value_len]
    return out


def encode_batched_accept_reply(paxos_id, version, acceptor, bnum, bcoord, slot_number, max_cp, request_id,
                                slots, req_ids) -> bytes:
    L = _lib()
    pid = paxos_id.encode("iso-8859-1")
    s = np.ascontiguousarray(slots, dtype=np.int32)
    q = np.ascontiguousarray(req_ids, dtype=np.int64)
    cap = 13 + len(pid) + 29 + 4 + 12 * len(s)
    buf = C.create_string_buffer(cap)
    n = L.gpx_wire_encode_batched_accept_reply(pid, C.c_uint32(len(pid)), C.c_int32(version), C.c_int32(acceptor),
                                               C.c_int32(bnum), C.c_int32(bcoord), C.c_int32(slot_number),
                                               C.c_int32(max_cp), C.c_int64(request_id), C.c_uint32(len(s)),
                                               s.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), buf,
                                               C.c_size_t(cap))
    assert n > 0
    return buf.raw[:n]


def decode_batched_accept_reply(b: bytes) -> dict:
    L = _lib()
    ver, acc, bn, bc, sn, mc, n = (C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32(),
                                   C.c_uint32())
    pid = C.create_string_buffer(128)
    pl = C.c_uint32()
    cap = max(1, len(b) // 12)
    slots = np.zeros(cap, np.int32)
    rids = np.zeros(cap, np.int64)
    rc = L.gpx_wire_decode_batched_accept_reply(b, C.c_size_t(len(b)), C.byref(ver), pid, C.byref(pl), C.byref(acc),
                                                C.byref(bn), C.byref(bc), C.byref(sn), C.byref(mc), C.byref(n),
                                                slots.ctypes.data_as(C.c_void_p), rids.ctypes.data_as(C.c_void_p),
                                                C.c_uint32(cap))
    if rc != 0:
        raise ValueError("malformed BATCHED_ACCEPT_REPLY")
    return dict(paxos_id=pid.raw[: pl.value].decode("iso-8859-1"), version=ver.value, acceptor=acc.value,
                bnum=bn.value, bcoord=bc.value, slot_number=sn.value, max_cp=mc.value,
                slots=slots[: n.value].tolist(), req_ids=rids[: n.value].tolist())


def encode_batched_commit(paxos_id, version, bnum, bcoord, median_cp, slots, group) -> bytes:
    L = _lib()
    pid = paxos_id.encode("iso-8859-1")
    s = np.ascontiguousarray(slots, dtype=np.int32)
    g = np.ascontiguousarray(group, dtype=np.int32)
    cap = 13 + len(pid) + 12 + 4 * (len(s) + len(g) + 2)
    buf = C.create_string_buffer(cap)
    n = L.gpx_wire_encode_batched_commit(pid, C.c_uint32(len(pid)), C.c_int32(version), C.c_int32(bnum),
                                         C.c_int32(bcoord), C.c_int32(median_cp), C.c_uint32(len(s)),
                                         s.ctypes.data_as(C.c_void_p), C.c_uint32(len(g)),
                                         g.ctypes.data_as(C.c_void_p), buf, C.c_size_t(cap))
    assert n > 0
    return buf.raw[:n]


def decode_batched_commit(b: bytes) -> dict:
    L = _lib()
    ver, bn, bc, mc, ns, ng = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_uint32(), C.c_uint32()
    pid = C.create_string_buffer(128)
    pl = C.c_uint32()
    cap = max(1, len(b) // 4)
    slots = np.zeros(cap, np.int32)
    group = np.zeros(cap, np.int32)
    rc = L.gpx_wire_decode_batched_commit(b, C.c_size_t(len(b)), C.byref(ver), pid, C.byref(pl), C.byref(bn),
                                          C.byref(bc), C.byref(mc), C.byref(ns), slots.ctypes.data_as(C.c_void_p),
                                          C.c_uint32(cap), C.byref(ng), group.ctypes.data_as(C.c_void_p),
                                          C.c_uint32(cap))
    if rc != 0:
        raise ValueError("malformed BATCHED_COMMIT")
    return dict(paxos_id=pid.raw[: pl.value].decode("iso-8859-1"), version=ver.value, bnum=bn.value, bcoord=bc.value,
                median_cp=mc.value, slots=slots[: ns.value].tolist(), group=group[: ng.value].tolist())


def journal_frame(packet: bytes) -> bytes:
    L = _lib()
    buf = C.create_string_buffer(len(packet) + 4)
    n = L.gpx_wire_journal_frame(packet, C.c_size_t(len(packet)), buf, C.c_size_t(len(packet) + 4))
    assert n == len(packet) + 4
    return buf.raw


def fuse_commits(decs: np.ndarray):
    """PaxosPacketBatcher.fuseBatchedCommits: (run_start, run_median_cp) of same-(gid,ballot) runs."""
    L = _lib()
    L.gpx_wire_fuse_commits.restype = C.c_uint32
    d = np.ascontiguousarray(decs, dtype=abi.decision_dtype)
    rs = np.zeros(max(len(d), 1), np.uint32)
    rm = np.zeros(max(len(d), 1), np.int32)
    k = L.gpx_wire_fuse_commits(C.c_uint32(len(d)), d.ctypes.data_as(C.c_void_p), rs.ctypes.data_as(C.c_void_p),
                                rm.ctypes.data_as(C.c_void_p))
    return rs[:k].copy(), rm[:k].copy()


# ---- phase-2 packets on the device (gpx_set_group_names, gpx_wire_decode_batch, gpx_wire_encode_*) -------------------
def pack_packets(packets: Sequence[bytes]):
    """(bytes arena, gpx_wire_ref[n]) for a list of packets"""
    refs = np.zeros(len(packets), dtype=abi.wire_ref_dtype)
    lens = np.array([len(p) for p in packets], dtype=np.uint64)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64) if len(packets) else lens
    refs["off"], refs["len"] = offs, lens
    arena = np.frombuffer(b"".join(packets), dtype=np.uint8) if packets else np.zeros(0, np.uint8)
    return np.ascontiguousarray(arena), refs


def unpack_packets(arena: np.ndarray, refs: np.ndarray) -> list:
    """[(gid, node, bytes)] of an encoder's output"""
    return [(int(r["gid"]), int(r["node"]), bytes(arena[int(r["off"]): int(r["off"]) + int(r["len"])])) for r in refs]


def set_group_names(engine, gids, names: Sequence[str]):
    """gpx_set_group_names: gids[k] is called names[k] (ISO-8859-1) at the version it was created / loaded with"""
    gids = np.ascontiguousarray(gids, dtype=np.uint32)
    enc = [s.encode("iso-8859-1") for s in names]
    lens = np.array([len(b) for b in enc], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint32) if len(enc) else lens
    arena = np.frombuffer(b"".join(enc) or b"\0", dtype=np.uint8)
    L = engine.L
    L.check(L.fn("set_group_names")(engine.handle, C.c_uint32(len(gids)), abi._ptr(gids), abi._ptr(arena),
                                    abi._ptr(offs), abi._ptr(lens)))


def _sized(engine, caps, size_types, alloc, call):
    """outputs = alloc(caps), then rc = call(outputs, sizes) with the sizes passed by reference (capacities in, sizes
    out); when an output is too small (GPX_ERANGE), both once more at the sizes the call reported -> (outputs, sizes)"""
    caps = [int(c) for c in caps]
    for _ in range(2):
        outs = alloc(caps)
        sz = [t(c) for t, c in zip(size_types, caps)]
        rc = call(outs, [C.byref(s) for s in sz])
        caps = [s.value for s in sz]
        if rc != abi.GPX_ERANGE:
            break
    engine.L.check(rc)
    return outs, tuple(caps)


def decode_batch(engine, packets: Sequence[bytes]):
    """gpx_wire_decode_batch -> (status[n], accepts, blob, replies, decisions); outputs grouped by gid"""
    L = engine.L
    arena, refs = pack_packets(packets)
    n = len(packets)
    status = np.zeros(max(n, 1), np.int32)
    (acc, blob, rep, dec), caps = _sized(  # sizes first: at capacity 0 any output is GPX_ERANGE
        engine, (0, 0, 0, 0), (C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32),
        lambda c: (np.zeros(max(c[0], 1), abi.accept_dtype), np.zeros(max(c[1], 16), np.uint8),
                   np.zeros(max(c[2], 1), abi.reply_dtype), np.zeros(max(c[3], 1), abi.decision_dtype)),
        lambda o, sz: L.fn("wire_decode_batch")(engine.handle, C.c_uint32(n), abi._ptr(arena), C.c_uint64(len(arena)),
                                                abi._ptr(refs), abi._ptr(status), abi._ptr(o[0]), sz[0],
                                                abi._ptr(o[1]), sz[1], abi._ptr(o[2]), sz[2], abi._ptr(o[3]), sz[3]))
    return (status[:n], acc[: caps[0]], blob[: caps[1]], rep[: caps[2]], dec[: caps[3]])


def _encode(engine, name, recs, dtype):
    L = engine.L
    recs = np.ascontiguousarray(recs, dtype=dtype)
    n = len(recs)
    rstatus = np.zeros(max(n, 1), np.uint8)
    (out, refs), caps = _sized(
        engine, (0, 0), (C.c_uint64, C.c_uint32),
        lambda c: (np.zeros(max(c[0], 1), np.uint8), np.zeros(max(c[1], 1), abi.wire_ref_dtype)),
        lambda o, sz: L.fn(name)(engine.handle, C.c_uint32(n), abi._ptr(recs), abi._ptr(rstatus), abi._ptr(o[0]),
                                 sz[0], abi._ptr(o[1]), sz[1]))
    return rstatus[:n], out[: caps[0]], refs[: caps[1]]


def encode_replies(engine, replies: np.ndarray):
    """gpx_wire_encode_replies over gpx_handle_accepts' output -> (rstatus[n], arena, refs)"""
    return _encode(engine, "wire_encode_replies", replies, abi.reply_dtype)


def encode_decisions(engine, decisions: np.ndarray):
    """gpx_wire_encode_decisions over gpx_handle_accept_replies' output -> (rstatus[n], arena, refs)"""
    return _encode(engine, "wire_encode_decisions", decisions, abi.decision_dtype)


# ---- the device-buffer forms (gpx_wire_*_device) over torch CUDA tensors ---------------------------------------------
# Records travel as uint8 tensors of shape [k, record bytes] (48 for accepts, 32 for replies and decisions, 16 for
# gpx_wire_ref); to_records() reads one as a numpy structured array.
DecodeOut = namedtuple("DecodeOut", "status accepts blob replies decisions sizes")
EncodeOut = namedtuple("EncodeOut", "rstatus out refs sizes")


def _dptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def stream_handle(stream=None):
    """the stream handle a device-form call runs on: `stream`, else torch's current stream.  torch's default stream is
    CUDA's legacy stream; it is handed over as cudaStreamLegacy, because NULL would mean the engine's own stream."""
    import torch
    h = (stream if stream is not None else torch.cuda.current_stream()).cuda_stream
    return C.c_void_p(h or 1)


def _on(stream):
    """allocate the outputs on the stream the call runs on"""
    import contextlib
    import torch
    return torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext()


def device_packets(packets: Sequence[bytes], device="cuda"):
    """the device-tensor form of a packet arena (pack_packets): (bytes uint8 [n_bytes], refs uint8 [n, 16])"""
    import torch
    arena, refs = pack_packets(packets)
    return (torch.from_numpy(arena.copy()).to(device),
            torch.from_numpy(refs.view(np.uint8).reshape(len(refs), 16)).to(device))


def to_records(t, dtype) -> np.ndarray:
    """a record tensor of the device forms as a numpy structured array (copied to the host)"""
    return np.ascontiguousarray(t.detach().cpu().numpy()).reshape(-1).view(dtype)


def decode_batch_device(engine, arena, refs, caps, stream=None) -> DecodeOut:
    """gpx_wire_decode_batch_device: the packets refs[n] (gpx_wire_ref rows) of the byte arena `arena`, both CUDA tensors
    (device_packets).  The outputs are allocated with caps = (accepts, blob bytes, replies, decisions); when one is too
    small (GPX_ERANGE) they are allocated again at the sizes the call reports and the call is repeated.  Returns views:
    status int32 [n], accepts [na, 48], blob [bytes], replies [nr, 32], decisions [nd, 32] -- grouped by gid, ready for
    gpx_accepts_device (n_chunks = 0), gpx_replies_device and gpx_decisions_device -- and the four host sizes, which a
    caller can hand to the next batch as its caps."""
    import torch
    n, dev = int(refs.shape[0]), refs.device
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        (acc, blob, rep, dec), caps = _sized(
            engine, caps, (C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32),
            lambda c: (torch.empty((max(c[0], 1), 48), dtype=torch.uint8, device=dev),
                       torch.empty(max(c[1], 16), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[2], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[3], 1), 32), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_decode_batch_device")(engine.handle, C.c_uint32(n), _dptr(arena),
                                                           C.c_uint64(arena.numel()), _dptr(refs), _dptr(status),
                                                           _dptr(o[0]), sz[0], _dptr(o[1]), sz[1], _dptr(o[2]), sz[2],
                                                           _dptr(o[3]), sz[3], st))
    return DecodeOut(status[:n], acc[: caps[0]], blob[: caps[1]], rep[: caps[2]], dec[: caps[3]], caps)


def _encode_device(engine, name, lead, n, dev, caps, stream) -> EncodeOut:
    import torch
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        rstatus = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        (out, refs), caps = _sized(
            engine, caps, (C.c_uint64, C.c_uint32),
            lambda c: (torch.empty(max(c[0], 1), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[1], 1), 16), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn(name)(engine.handle, *lead, _dptr(rstatus), _dptr(o[0]), sz[0], _dptr(o[1]), sz[1], st))
    return EncodeOut(rstatus[:n], out[: caps[0]], refs[: caps[1]], caps)


def encode_replies_device(engine, replies, n: int, caps, stream=None) -> EncodeOut:
    """gpx_wire_encode_replies_device over the first n records of `replies` (a CUDA tensor in gpx_accepts_device's
    layout, n = n_lanes x the ACCEPTs handled).  caps = (packet bytes, packets); GPX_ERANGE as in decode_batch_device.
    Returns rstatus uint8 [n], the packet arena, refs [k, 16] and the two host sizes."""
    return _encode_device(engine, "wire_encode_replies_device", (C.c_uint32(n), _dptr(replies)), n,
                          replies.device, caps, stream)


def encode_decisions_device(engine, decisions, n_ptr: Optional[int], n_max: int, caps, stream=None) -> EncodeOut:
    """gpx_wire_encode_decisions_device: the record count is read on the device at address n_ptr (e.g. the
    n_decisions word of the gpx_dev_ctl that gpx_replies_device counted into), at most n_max; None = n_max.
    rstatus [n_max] is written only below that count."""
    return _encode_device(engine, "wire_encode_decisions_device",
                          (_dptr(decisions), C.c_void_p(n_ptr) if n_ptr else None, C.c_uint32(n_max)), n_max,
                          decisions.device, caps, stream)


JsonOut = namedtuple("JsonOut", "status members replies decisions sizes")


def decode_json_device(engine, arena, refs, caps, stream=None) -> JsonOut:
    """gpx_wire_decode_json_device: the JSON packets refs[n] of `arena` (device_packets; the refs' node column names
    the node that received each packet) -- BATCHED_PAXOS_PACKET wrappers and bare ACCEPT_REPLY / BATCHED_ACCEPT_REPLY /
    BATCHED_COMMIT packets.  caps = (members, replies, decisions); GPX_ERANGE as in decode_batch_device.  Returns
    status int32 [n], members [m, 16] (abi.wire_member_dtype), replies [nr, 32] and decisions [nd, 32] grouped by gid
    (gpx_replies_device's and gpx_decisions_device's input form) and the three host sizes."""
    import torch
    n, dev = int(refs.shape[0]), refs.device
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        (mem, rep, dec), caps = _sized(
            engine, caps, (C.c_uint32, C.c_uint32, C.c_uint32),
            lambda c: (torch.empty((max(c[0], 1), 16), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[1], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[2], 1), 32), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_decode_json_device")(engine.handle, C.c_uint32(n), _dptr(arena),
                                                          C.c_uint64(arena.numel()), _dptr(refs), _dptr(status),
                                                          _dptr(o[0]), sz[0], _dptr(o[1]), sz[1], _dptr(o[2]), sz[2],
                                                          st))
    return JsonOut(status[:n], mem[: caps[0]], rep[: caps[1]], dec[: caps[2]], caps)


JsonEncodeOut = namedtuple("JsonEncodeOut", "rstatus_replies rstatus_decisions out refs sizes")


def encode_json_device(engine, replies, n_replies: int, decisions, n_dec_ptr: Optional[int], n_dec_max: int, caps,
                       wrap_bytes: int = 0, stream=None) -> JsonEncodeOut:
    """gpx_wire_encode_json_device: the first n_replies records of `replies` (gpx_accepts_device's layout) and the
    decisions (count read on the device at address n_dec_ptr, at most n_dec_max; None = n_dec_max) as the JSON a loaded
    Java node sends -- BATCHED_PAXOS_PACKET wrappers of at most wrap_bytes (0 = 4 MiB) per recipient set, each NACK a
    bare ACCEPT_REPLY.  Either tensor may be None when its count is 0.  caps = (packet bytes, refs); GPX_ERANGE as in
    decode_batch_device.  Returns both rstatus arrays (uint8), the packet arena, refs [k, 16] (a wrapper's gid column
    is its sending lane) and the two host sizes."""
    import torch
    dev = (replies if replies is not None else decisions).device
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        rr = torch.empty(max(n_replies, 1), dtype=torch.uint8, device=dev)
        rd = torch.empty(max(n_dec_max, 1), dtype=torch.uint8, device=dev)
        (out, refs), caps = _sized(
            engine, caps, (C.c_uint64, C.c_uint32),
            lambda c: (torch.empty(max(c[0], 1), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[1], 1), 16), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_encode_json_device")(engine.handle, C.c_uint32(n_replies), _dptr(replies),
                                                          _dptr(decisions), C.c_void_p(n_dec_ptr) if n_dec_ptr else None,
                                                          C.c_uint32(n_dec_max), _dptr(rr), _dptr(rd),
                                                          C.c_uint64(wrap_bytes), _dptr(o[0]), sz[0], _dptr(o[1]),
                                                          sz[1], st))
    return JsonEncodeOut(rr[:n_replies], rd[:n_dec_max], out[: caps[0]], refs[: caps[1]], caps)


JsonSweepOut = namedtuple("JsonSweepOut", "rstatus_replies rstatus_decisions rstatus_reqs out refs sizes")


def encode_json_sweep_device(engine, replies, n_replies: int, decisions, n_dec_ptr: Optional[int], n_dec_max: int,
                             reqs, meta, n_reqs: int, status, payload, down_nodes: Sequence[int], caps,
                             wrap_bytes: int = 0, stream=None) -> JsonSweepOut:
    """gpx_wire_encode_json_sweep_device: encode_json_device's replies and decisions, and the forwarded requests among
    the first n_reqs of reqs / meta (encode_forwards_device's inputs), as one sweep -- a forward of one request is a
    REQUEST member of the wrapper to its coordinator, any other forward a lone REQUEST packet.  Any tensor may be None
    when its count is 0.  caps = (packet bytes, refs); GPX_ERANGE as in decode_batch_device.  Returns the three rstatus
    arrays (uint8; rstatus_reqs is encode_forwards_device's), the packet arena, refs [k, 16] (bare NACKs, lone
    REQUEST packets, wrappers) and the two host sizes."""
    import torch
    dev = next(t for t in (replies, decisions, reqs) if t is not None).device
    down = np.ascontiguousarray(list(down_nodes) or [0], dtype=np.int32)
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        rr = torch.empty(max(n_replies, 1), dtype=torch.uint8, device=dev)
        rd = torch.empty(max(n_dec_max, 1), dtype=torch.uint8, device=dev)
        rq = torch.empty(max(n_reqs, 1), dtype=torch.uint8, device=dev)
        (out, refs), caps = _sized(
            engine, caps, (C.c_uint64, C.c_uint32),
            lambda c: (torch.empty(max(c[0], 1), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[1], 1), 16), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_encode_json_sweep_device")(
                engine.handle, C.c_uint32(n_replies), _dptr(replies), _dptr(decisions),
                C.c_void_p(n_dec_ptr) if n_dec_ptr else None, C.c_uint32(n_dec_max), _dptr(reqs), _dptr(meta),
                C.c_uint32(n_reqs), _dptr(status), _dptr(payload), C.c_uint32(len(down_nodes)),
                down.ctypes.data_as(C.c_void_p), _dptr(rr), _dptr(rd), _dptr(rq), C.c_uint64(wrap_bytes),
                _dptr(o[0]), sz[0], _dptr(o[1]), sz[1], st))
    return JsonSweepOut(rr[:n_replies], rd[:n_dec_max], rq[:n_reqs], out[: caps[0]], refs[: caps[1]], caps)


# ---- the coordinator's side: REQUEST packets -> proposals -> ACCEPT packets, on the device ---------------------------
RequestsOut = namedtuple("RequestsOut", "status reqs meta payload sizes")


def req_meta(r: Request) -> np.ndarray:
    """the gpx_wire_req_meta of a Request: the wire fields a gpx_request_rec does not keep"""
    m = np.zeros(1, abi.req_meta_dtype)
    for name, a in (("client", r.client), ("listen", r.listen)):
        if a is not None and a[1]:
            m[name + "_ip"][0] = [int(x) for x in a[0].split(".")]
            m[name + "_port"] = a[1]
    m["forward_count"], m["entry_time"] = r.forward_count, r.entry_time
    m["flags"] = (abi.RM_RETURN_VALUE if r.should_return else 0) | (abi.RM_BROADCASTED if r.broadcasted else 0)
    return m[0]


def decode_requests_device(engine, arena, refs, now_ms: int, caps, stream=None) -> RequestsOut:
    """gpx_wire_decode_requests_device: the REQUEST packets refs[n] of `arena` (device_packets; the refs' node column
    names the node that received each packet).  caps = (requests, payload bytes); GPX_ERANGE as in decode_batch_device.
    Returns status int32 [n], reqs [k, 32] and meta [k, 32] (grouped by gid, gpx_propose_device's input form), the
    payload arena and the two host sizes."""
    import torch
    n, dev = int(refs.shape[0]), refs.device
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        (reqs, meta, pay), caps = _sized(
            engine, caps, (C.c_uint32, C.c_uint64),
            lambda c: (torch.empty((max(c[0], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[0], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty(max(c[1], 16), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_decode_requests_device")(engine.handle, C.c_uint32(n), _dptr(arena),
                                                              C.c_uint64(arena.numel()), _dptr(refs), C.c_int64(now_ms),
                                                              _dptr(status), _dptr(o[0]), _dptr(o[1]), sz[0],
                                                              _dptr(o[2]), sz[1], st))
    return RequestsOut(status[:n], reqs[: caps[0]], meta[: caps[0]], pay[: caps[1]], caps)


def propose_device_heads(engine, reqs, n: int, payload, payload_bytes: int, status, accepts, heads, ctl, stream=None):
    """gpx_propose_device_heads over CUDA tensors: the ACCEPTs at `accepts` ([n, 48]), counted in ctl (gpx_dev_ctl,
    zeroed by the caller), and heads [n] uint32: the request that starts each ACCEPT, 0xffffffff for a VOID filler"""
    L = engine.L
    L.check(L.fn("propose_device_heads")(engine.handle, _dptr(reqs), _dptr(payload), C.c_uint64(payload_bytes),
                                         C.c_uint32(n), _dptr(status), _dptr(accepts), _dptr(heads), _dptr(ctl),
                                         stream_handle(stream)))


def encode_accepts_device(engine, accepts, n_ptr: Optional[int], n_max: int, heads, reqs, meta, n_reqs: int, payload,
                          caps, stream=None) -> EncodeOut:
    """gpx_wire_encode_accepts_device: AcceptPackets of the ACCEPTs (count read on the device at address n_ptr, e.g.
    the n_accepts word of the gpx_dev_ctl propose_device_heads counted into, at most n_max; None = n_max), their
    requests read at heads[k] of reqs / meta / payload.  caps = (packet bytes, packets); GPX_ERANGE as in
    decode_batch_device."""
    return _encode_device(engine, "wire_encode_accepts_device",
                          (_dptr(accepts), C.c_void_p(n_ptr) if n_ptr else None, C.c_uint32(n_max), _dptr(heads),
                           _dptr(reqs), _dptr(meta), C.c_uint32(n_reqs), _dptr(payload)), n_max, accepts.device, caps,
                          stream)


# ---- forwarding: a non-coordinator's REQUEST packets, and a Java peer's forwards in JSON wrappers ---------------------
def encode_forwards_device(engine, reqs, meta, n: int, status, payload, down_nodes: Sequence[int], caps,
                           stream=None) -> EncodeOut:
    """gpx_wire_encode_forwards_device: the forwarded requests among the first n of reqs / meta (propose_device's input,
    with its statuses and payload arena) as REQUEST packets addressed to their coordinators; down_nodes are the nodes
    the host takes for down.  caps = (packet bytes, packets); GPX_ERANGE as in decode_batch_device.  Returns rstatus
    uint8 [n] (WE_SENT, WE_VOID, WE_ELECT, WE_NO_NAME), the packet arena, refs [k, 16] in request order and the two host
    sizes."""
    down = np.ascontiguousarray(list(down_nodes) or [0], dtype=np.int32)
    return _encode_device(engine, "wire_encode_forwards_device",
                          (_dptr(reqs), _dptr(meta), C.c_uint32(n), _dptr(status), _dptr(payload),
                           C.c_uint32(len(down_nodes)), down.ctypes.data_as(C.c_void_p)), n, reqs.device, caps, stream)


def decode_json_requests_device(engine, arena, refs, members, n_members: int, now_ms: int, caps,
                                stream=None) -> RequestsOut:
    """gpx_wire_decode_json_requests_device: the REQUEST members among the first n_members rows of `members` (what
    decode_json_device returned for the same arena and refs; the refs' node column names the receiving node).
    caps = (requests, payload bytes); GPX_ERANGE as in decode_batch_device.  Returns status int32 [n_members] (the
    decoded members' statuses, the others copied), reqs [k, 32] and meta [k, 32] grouped by gid (propose_device's input
    form, client = the member index), the payload arena and the two host sizes."""
    import torch
    n, dev = int(n_members), members.device
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        (reqs, meta, pay), caps = _sized(
            engine, caps, (C.c_uint32, C.c_uint64),
            lambda c: (torch.empty((max(c[0], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[0], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty(max(c[1], 16), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_decode_json_requests_device")(
                engine.handle, C.c_uint32(n), _dptr(arena), C.c_uint64(arena.numel()), _dptr(refs),
                C.c_uint32(int(refs.shape[0])), _dptr(members), C.c_int64(now_ms), _dptr(status), _dptr(o[0]),
                _dptr(o[1]), sz[0], _dptr(o[2]), sz[1], st))
    return RequestsOut(status[:n], reqs[: caps[0]], meta[: caps[0]], pay[: caps[1]], caps)


# ---- a client's own requests: bare JSON REQUEST packets, addressed by their connection ---------------------------------
def wire_peers(peers) -> np.ndarray:
    """[(sender, receiver)] -> abi.wire_peer_dtype rows; an address is (ip, port) or None (port 0: unknown)"""
    out = np.zeros(len(peers), abi.wire_peer_dtype)
    for k, (snd, rcv) in enumerate(peers):
        for pre, a in (("sender", snd), ("receiver", rcv)):
            if a is not None:
                out[k][pre + "_ip"] = [int(x) for x in a[0].split(".")]
                out[k][pre + "_port"] = a[1]
    return out


def decode_client_requests_device(engine, arena, refs, peers, now_ms: int, caps, stream=None) -> RequestsOut:
    """gpx_wire_decode_client_requests_device: the bare JSON REQUEST packets a client sends, refs[n] of `arena` (the
    refs' node column names the receiving node), peers [n, 16] (abi.wire_peer_dtype rows on the device: each packet's
    connection, the fallback client and listen address; None: no fallback).  caps = (requests, payload bytes);
    GPX_ERANGE as in decode_batch_device.  Returns status int32 [n] (byteified packets and other JSON types
    WS_UNHANDLED), reqs [k, 32] and meta [k, 32] grouped by gid (propose_device's input form, client = the packet
    index), the payload arena and the two host sizes."""
    import torch
    n, dev = int(refs.shape[0]), refs.device
    L, st = engine.L, stream_handle(stream)
    with _on(stream):
        status = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
        (reqs, meta, pay), caps = _sized(
            engine, caps, (C.c_uint32, C.c_uint64),
            lambda c: (torch.empty((max(c[0], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty((max(c[0], 1), 32), dtype=torch.uint8, device=dev),
                       torch.empty(max(c[1], 16), dtype=torch.uint8, device=dev)),
            lambda o, sz: L.fn("wire_decode_client_requests_device")(
                engine.handle, C.c_uint32(n), _dptr(arena), C.c_uint64(arena.numel()), _dptr(refs),
                _dptr(peers), C.c_int64(now_ms), _dptr(status), _dptr(o[0]),
                _dptr(o[1]), sz[0], _dptr(o[2]), sz[1], st))
    return RequestsOut(status[:n], reqs[: caps[0]], meta[: caps[0]], pay[: caps[1]], caps)
