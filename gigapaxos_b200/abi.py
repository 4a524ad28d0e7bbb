"""ctypes / numpy mirror of include/gpx.h (the C ABI of the engine).

Everything here is plumbing: record dtypes, the config/row structs and a thin `Engine`
wrapper whose methods are 1:1 with the C entry points.  The library path and symbol
prefix are parameters so that the test-suite can drive its CPU checker (own prefix)
through the very same wrapper; nothing in this package ever loads the oracle.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import namedtuple
from typing import Optional

import numpy as np

GPX_ABI_VERSION = 2
GPX_MAX_GROUP_SIZE = 16
GPX_MAX_LANES = 8
GPX_MAX_WINDOW = 8

# return codes
GPX_OK, GPX_EINVAL, GPX_ENOMEM, GPX_ECUDA, GPX_ENOGPU, GPX_ERANGE, GPX_EIO, GPX_EAGAIN = 0, -1, -2, -3, -4, -5, -6, -7
GPX_ENOENT = -8  # gpx_log_frame_device: requests or names the frames need are missing (listed)
# PaxosAcceptor.STATES ordinals
ST_RECOVERY, ST_ACTIVE_1, ST_ACTIVE_2, ST_STOPPED, ST_FREE = 0, 1, 2, 3, 255
# record flags
F_STOP, F_VOID, F_ACCEPT, F_DECISION, F_META, F_CKPT, F_LOGGED, F_NACK, F_EXTRA = (
    0x1, 0x2, 0x4, 0x8, 0x10, 0x20, 0x40, 0x80, 0x100)
# request status codes
RS_BATCHED, RS_FORWARD, RS_REFUSED_STOP, RS_BACKPRESSURE, RS_DROPPED, RS_PREACTIVE, RS_NOCOORD = (
    -1, -2, -3, -4, -5, -6, -7)
INIT_BATCH, INIT_DEFAULT = 0, 1
GF_OVERFLOW, GF_NEEDS_SYNC, GF_NOT_CAUGHT_UP = 1, 2, 4  # gpx_get_group_flags bits
PATCH_SET_BALLOT, PATCH_JUMP_SLOT, PATCH_SET_STATE, PATCH_INSTALL_COORD, PATCH_RESIGN_COORD, PATCH_SET_GC = (
    1, 2, 3, 4, 5, 6)
PATCH_SET_NODE_SLOT = 7
SEG_MAGIC = 0x53585047

request_dtype = np.dtype([("gid", "<u4"), ("flags", "<u4"), ("req_id", "<i8"), ("payload_off", "<u4"),
                          ("payload_len", "<u4"), ("entry_node", "<i4"), ("client", "<u4")])
pvalue_fields = [("gid", "<u4"), ("slot", "<i4"), ("bnum", "<i4"), ("bcoord", "<i4"), ("median_cp", "<i4"),
                 ("flags", "<u2"), ("dst_mask", "<u2"), ("req_id", "<i8")]
decision_dtype = np.dtype(pvalue_fields)
accept_dtype = np.dtype(pvalue_fields + [("payload_off", "<u4"), ("payload_len", "<u4"), ("nreq", "<u4"),
                                         ("sender", "<i4")])
reply_dtype = np.dtype([("gid", "<u4"), ("slot", "<i4"), ("bnum", "<i4"), ("bcoord", "<i4"), ("max_cp", "<i4"),
                        ("who", "<u4"), ("req_id", "<i8")])
exec_dtype = np.dtype([("gid", "<u4"), ("slot", "<i4"), ("req_id", "<i8"), ("payload_off", "<u4"), ("flags", "<u4")])
batch_ent_dtype = np.dtype([("req_id", "<i8"), ("len", "<u4"), ("flags", "<u4")])
wire_ref_dtype = np.dtype([("off", "<u4"), ("len", "<u4"), ("gid", "<u4"), ("node", "<i4")])  # gpx_wire_ref
# per-packet status of gpx_wire_decode_batch, per-record outcome of gpx_wire_encode_*
WS_OK, WS_UNKNOWN_NAME, WS_VERSION, WS_MALFORMED, WS_UNHANDLED, WS_NOT_LOCAL = 0, 1, 2, 3, 4, 5
WE_SENT, WE_VOID, WE_LOCAL, WE_NACK, WE_NO_NAME = 0, 1, 2, 3, 4
WE_BAD_HEAD = 5  # gpx_wire_encode_accepts_device: the ACCEPT's head request is out of range or of another group
WE_ELECT = 6  # gpx_wire_encode_forwards_device: the host runs for coordinator instead of forwarding
# gpx_wire_req_meta: the RequestPacket wire fields a gpx_request_rec does not keep (gpx_wire_decode_requests_device)
RM_RETURN_VALUE, RM_BROADCASTED = 1, 2
req_meta_dtype = np.dtype([("client_ip", "u1", (4,)), ("client_port", "<u2"), ("listen_port", "<u2"),
                           ("listen_ip", "u1", (4,)), ("forward_count", "<i4"), ("entry_time", "<i8"),
                           ("flags", "<u4"), ("pad", "<u4")])
assert req_meta_dtype.itemsize == 32
# gpx_rc_key: one executed client request for the response cache (gpx_response_cache_put_device)
rc_key_dtype = np.dtype([("gid", "<u4"), ("handle", "<i4"), ("req_id", "<i8"), ("client_ip", "u1", (4,)),
                         ("client_port", "<u2"), ("pad", "<u2")])
assert rc_key_dtype.itemsize == 24
# gpx_wire_peer: the connection a client's packet came in on (gpx_wire_decode_client_requests_device); port 0 = unknown
wire_peer_dtype = np.dtype([("sender_ip", "u1", (4,)), ("sender_port", "<u2"), ("receiver_port", "<u2"),
                            ("receiver_ip", "u1", (4,)), ("pad", "<u4")])
assert wire_peer_dtype.itemsize == 16
# gpx_wire_member: one member of a JSON packet (gpx_wire_decode_json_device)
wire_member_dtype = np.dtype([("pkt", "<u4"), ("off", "<u4"), ("len", "<u4"), ("status", "<i4")])
# gpx_wire_encode_json_device: a wrapper's default and largest size, its head + tail, the largest member object
GPX_JSON_WRAP_BYTES, GPX_JSON_WRAP_OVERHEAD, GPX_JSON_MAX_MEMBER = 4 << 20, 34, 65536
accepted_pvalue_dtype = np.dtype([("slot", "<i4"), ("bnum", "<i4"), ("bcoord", "<i4"), ("frame_ref", "<u4"),
                                  ("req_id", "<i8"), ("payload_len", "<u4"), ("flags", "<u4")])
prepare_reply_dtype = np.dtype([("gid", "<u4"), ("first_slot", "<i4"), ("bnum", "<i4"), ("bcoord", "<i4"), ("who", "<u4"),
                                ("n_accepted", "<u4"), ("reserved", "<i8"),
                                ("accepted", accepted_pvalue_dtype, (GPX_MAX_WINDOW,))])
assert prepare_reply_dtype.itemsize == 32 + 32 * GPX_MAX_WINDOW
F_PREPARE, F_FROM_LOG, F_MORE = 0x200, 0x400, 0x800
# phase 1b (gpx_handle_prepare_replies)
GPX_MAX_CARRY, GPX_MAX_PLAN = 32, 16
EL_WAITING, EL_MAJORITY, EL_PREEMPTED, EL_DROPPED, EL_OVERFLOW = 0, 1, 2, 3, 4
CO_NOOP, CO_PVALUE, CO_STOP_NEW = 0, 1, 2
ELF_STOP_ORDER = 1
election_dtype = np.dtype([("gid", "<u4"), ("lane", "<u4"), ("bnum", "<i4"), ("bcoord", "<i4"), ("slot", "<i4"),
                           ("first_reply", "<u4"), ("n_replies", "<u4"), ("reserved", "<u4")])
carryover_dtype = np.dtype([("slot", "<i4"), ("kind", "<u4"), ("src_reply", "<u4"), ("reserved", "<u4"),
                            ("pv", accepted_pvalue_dtype)])
election_out_dtype = np.dtype([("gid", "<u4"), ("verdict", "<i4"), ("next_slot", "<i4"), ("n_plan", "<u2"),
                               ("flags", "<u2"), ("node_slots", "<i4", (GPX_MAX_GROUP_SIZE,)),
                               ("plan", carryover_dtype, (GPX_MAX_PLAN + 1,))])
assert election_dtype.itemsize == 32 and carryover_dtype.itemsize == 48 and election_out_dtype.itemsize == 896
# gpx_log_find
GPX_LOG_SPAN = 16
log_want_dtype = np.dtype([("gid", "<u4"), ("min_slot", "<i4"), ("n_slots", "<u4"), ("reserved", "<u4")])
log_hit_dtype = np.dtype([("decision", decision_dtype), ("accept", accept_dtype), ("blob_pos", "<u8"), ("reserved", "<u8")])
assert log_want_dtype.itemsize == 16 and log_hit_dtype.itemsize == 96
log_range_dtype = np.dtype([("pos", "<u8"), ("len", "<u4"), ("dst_off", "<u4")])
# gpx_log_frame_device: the caller's table of the RequestPacket fields the ring does not hold, and what a call lacks
journal_req_dtype = np.dtype([("gid", "<u4"), ("entry_node", "<i4"), ("req_id", "<i8"), ("entry_time", "<i8")])
journal_miss_dtype = np.dtype([("gid", "<u4"), ("kind", "<u4"), ("req_id", "<i8")])
assert journal_req_dtype.itemsize == 24 and journal_miss_dtype.itemsize == 16
# gpx_journal_compact_device: what the call did to each file
journal_file_dtype = np.dtype([("status", "<u4"), ("kept", "<u4"), ("dropped", "<u4"), ("unresolved", "<u4"),
                               ("out_off", "<u4"), ("out_bytes", "<u4")])
assert journal_file_dtype.itemsize == 24
missing_dtype = np.dtype([("gid", "<u4"), ("slot", "<i4"), ("max_decision_slot", "<i4"), ("n_missing", "<u2"),
                          ("missing_too_much", "u1"), ("flags", "u1"), ("missing", "<i4", (GPX_MAX_WINDOW,))])
assert missing_dtype.itemsize == 48
exec_sum_dtype = np.dtype([("slot", "<i4"), ("lane_mask", "u1"), ("flags", "u1"), ("nreq", "<u2")])
ROUND_COMPACT = 1
ROUND_PACKED_REQS = 2
request_packed_dtype = np.dtype([("gid", "<u4"), ("payload_len", "<u2"), ("flags", "<u2"), ("req_id", "<i8")])
PIPE_DEPTH = 4
seg_hdr_dtype = np.dtype([("magic", "<u4"), ("type", "<u2"), ("lane", "<u2"), ("n_slots", "<u4"), ("n_valid", "<u4"),
                          ("payload_bytes", "<u8"), ("seq", "<u8"), ("ring_off", "<u8"), ("rec_bytes", "<u4"),
                          ("reserved", "<u4", (5,))])
row_dtype = np.dtype([("gid", "<u4"), ("lane", "<u4"), ("version", "<i4"), ("acc_slot", "<i4"), ("acc_bnum", "<i4"),
                      ("acc_bcoord", "<i4"), ("acc_gc_slot", "<i4"), ("state", "<i4"), ("coord_exists", "<i4"),
                      ("coord_active", "<i4"), ("coord_bnum", "<i4"), ("coord_bcoord", "<i4"),
                      ("next_proposal_slot", "<i4"), ("n_members", "<i4"), ("members", "<i4", (16,)),
                      ("node_slots", "<i4", (16,)), ("name_hash", "<i4")])
group_desc_dtype = np.dtype([("gid", "<u4"), ("version", "<i4"), ("name_hash", "<i4"), ("n_members", "<i4"),
                             ("members", "<i4", (16,)), ("init_mode", "<i4")])
patch_dtype = np.dtype([("gid", "<u4"), ("lane", "<u4"), ("op", "<i4"), ("a", "<i4"), ("b", "<i4"), ("c", "<i4"),
                        ("d", "<i4"), ("reserved", "<i4")])

assert request_dtype.itemsize == 32 and decision_dtype.itemsize == 32 and accept_dtype.itemsize == 48
assert reply_dtype.itemsize == 32 and exec_dtype.itemsize == 24 and seg_hdr_dtype.itemsize == 64
assert row_dtype.itemsize == 56 + 128 + 4 and group_desc_dtype.itemsize == 84 and patch_dtype.itemsize == 32

COUNTER_NAMES = ["accepts_handled", "accepts_acked", "accepts_nacked", "accepts_logged", "accepts_dropped",
                 "replies_handled", "replies_ignored", "preempted", "coordinators_resigned", "decisions_made",
                 "decisions_handled", "decisions_dropped", "placeholders", "executed", "stops_executed",
                 "checkpoints_due", "proposals", "requests_batched", "requests_rejected", "window_overflow",
                 "kernel_launches"]


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("device", C.c_int32), ("max_groups", C.c_uint32), ("n_lanes", C.c_uint32),
        ("lane_node", C.c_int32 * GPX_MAX_LANES), ("window", C.c_uint32), ("max_group_size", C.c_uint32),
        ("log_ring_bytes", C.c_uint64), ("max_batch_recs", C.c_uint32), ("max_batch_payload", C.c_uint64),
        ("batching_enabled", C.c_int32), ("max_batch_size", C.c_int32), ("max_batch_bytes", C.c_int64),
        ("request_size_estimate", C.c_int32), ("checkpoint_interval", C.c_int32), ("cpi_noise", C.c_double),
        ("gc_majority_executed", C.c_int32), ("log_meta_decisions", C.c_int32), ("journaling_enabled", C.c_int32),
        ("log_backpressure", C.c_int32),
        ("reserved", C.c_int32 * 7),
    ]


class Counters(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in COUNTER_NAMES] + [("reserved", C.c_uint64 * 7)]


class KernelTimes(C.Structure):
    _fields_ = [("propose_ms", C.c_double), ("accept_ms", C.c_double), ("tally_ms", C.c_double),
                ("commit_ms", C.c_double), ("launches", C.c_uint64)]


class DevRoundBufs(C.Structure):
    _fields_ = [("reqs", C.c_void_p), ("payload", C.c_void_p), ("payload_bytes", C.c_uint64), ("n", C.c_uint32),
                ("status", C.c_void_p), ("exec", C.c_void_p)]


class RoundIO(C.Structure):
    _fields_ = [("n", C.c_uint32), ("flags", C.c_uint32), ("reqs", C.c_void_p), ("payload", C.c_void_p),
                ("payload_bytes", C.c_uint64), ("status", C.c_void_p), ("exec", C.c_void_p), ("sum", C.c_void_p),
                ("extra", C.c_void_p), ("extra_cap", C.c_uint32)]


SPREAD_MAX_NODES = 8
SPREAD_GRAPH = 1
SPREAD_P2P = 2


class SpreadConfig(C.Structure):
    """gpx_spread_config (include/gpx.h)"""
    _fields_ = [("n_nodes", C.c_uint32), ("node_ids", C.c_int32 * SPREAD_MAX_NODES),
                ("cap", (C.c_uint32 * SPREAD_MAX_NODES) * SPREAD_MAX_NODES), ("blob_per_rec", C.c_uint32),
                ("max_reqs", C.c_uint32), ("flags", C.c_uint32), ("reserved", C.c_uint32 * 8)]


class SpreadPlan(C.Structure):
    """gpx_spread_plan"""
    _U64x3 = (C.c_uint64 * SPREAD_MAX_NODES) * 3
    _fields_ = [("n_nodes", C.c_uint32), ("rank", C.c_uint32), ("send_off", _U64x3), ("send_bytes", _U64x3),
                ("recv_off", _U64x3), ("recv_bytes", _U64x3), ("vbase", C.c_uint32 * SPREAD_MAX_NODES),
                ("vtotal", C.c_uint32), ("blob_off", C.c_uint64 * SPREAD_MAX_NODES), ("blob_vtotal", C.c_uint64),
                ("arena_bytes", C.c_uint64)]


class SpreadIO(C.Structure):
    """gpx_spread_io: device pointers of one node's round"""
    _fields_ = [("reqs", C.c_void_p), ("payload", C.c_void_p), ("payload_bytes", C.c_uint64), ("n", C.c_uint32),
                ("reserved", C.c_uint32), ("status", C.c_void_p), ("exec", C.c_void_p), ("extra", C.c_void_p),
                ("extra_cap", C.c_uint32), ("reserved2", C.c_uint32), ("ctl", C.c_void_p)]


class GpxError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"gpx error {code}: {msg}")
        self.code = code


def who(acc_idx: int, dst_idx: int, flags: int = 0) -> int:
    return (acc_idx & 0xFF) | ((dst_idx & 0xFF) << 8) | ((flags & 0xFFFF) << 16)


def who_acc(w):
    return w & 0xFF


def who_dst(w):
    return (w >> 8) & 0xFF


def who_flags(w):
    return w >> 16


def java_string_hash(s: str) -> int:
    """java.lang.String.hashCode() for ISO-8859-1 / BMP strings."""
    h = 0
    for ch in s:
        h = (31 * h + ord(ch)) & 0xFFFFFFFF
    return h - (1 << 32) if h >= (1 << 31) else h


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Library:
    """A loaded C-ABI library (CUDA engine or, in tests, the oracle) with a symbol prefix."""

    def __init__(self, path: str, prefix: str = "gpx_"):
        if not os.path.exists(path):
            raise FileNotFoundError(
                f"{path} not found: build it with `python -m gigapaxos_b200.build` (there is no CPU fallback)")
        self.path, self.prefix = path, prefix
        self.lib = C.CDLL(path)
        self.fn("last_error").restype = C.c_char_p
        self.fn("build_info").restype = C.c_char_p

    def fn(self, name: str):
        return getattr(self.lib, self.prefix + name)

    def has(self, name: str) -> bool:
        return hasattr(self.lib, self.prefix + name)

    def last_error(self) -> str:
        return (self.fn("last_error")() or b"").decode()

    def build_info(self) -> str:
        return self.fn("build_info")().decode()

    def journal_index(self, buf: bytes, base: int = 0) -> np.ndarray:
        """gpx_journal_index: base + the offset of every whole frame of one journal file's bytes (uint32)"""
        cap = len(buf) // 4 + 1
        starts = np.zeros(cap, np.uint32)
        n, end = C.c_uint32(0), C.c_uint64(0)
        self.check(self.fn("journal_index")(C.c_char_p(bytes(buf)), C.c_uint64(len(buf)), C.c_uint32(base),
                                            _ptr(starts), C.c_uint32(cap), C.byref(n), C.byref(end)))
        return starts[: n.value]

    def config_defaults(self) -> Config:
        cfg = Config()
        self.fn("config_defaults")(C.byref(cfg))
        return cfg

    def check(self, rc: int):
        if rc != 0:
            raise GpxError(rc, self.last_error())


LogFrames = namedtuple("LogFrames", "rc from_ frames missing sizes")
JournalCompact = namedtuple("JournalCompact", "rc out files bad sizes")


class Engine:
    """1:1 wrapper over the gpx_* entry points.  Arrays are numpy structured arrays."""

    def __init__(self, library: Library, cfg: Config):
        self.L = library
        self.cfg = cfg
        self.n_lanes = int(cfg.n_lanes)
        self._h = C.c_void_p()
        self._inflight = {}
        library.check(library.fn("engine_create")(C.byref(cfg), C.byref(self._h)))

    def close(self):
        if self._h:
            self.L.fn("engine_destroy")(self._h)
            self._h = C.c_void_p()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    # ---- groups -------------------------------------------------------------------
    def create_groups(self, descs: np.ndarray):
        descs = np.ascontiguousarray(descs, dtype=group_desc_dtype)
        self.L.check(self.L.fn("create_groups")(self._h, C.c_uint32(len(descs)), _ptr(descs)))

    def destroy_groups(self, gids):
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        self.L.check(self.L.fn("destroy_groups")(self._h, C.c_uint32(len(gids)), _ptr(gids)))

    def dump_rows(self, gids, lane: int) -> np.ndarray:
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        out = np.zeros(len(gids), dtype=row_dtype)
        self.L.check(self.L.fn("dump_rows")(self._h, C.c_uint32(len(gids)), _ptr(gids), C.c_uint32(lane), _ptr(out)))
        return out

    def load_rows(self, rows: np.ndarray):
        rows = np.ascontiguousarray(rows, dtype=row_dtype)
        self.L.check(self.L.fn("load_rows")(self._h, C.c_uint32(len(rows)), _ptr(rows)))

    def log_find(self, lane: int, wants: np.ndarray, from_: int = 0) -> np.ndarray:
        """The journal's index as a scan (gpx_log_find): per want (gid, min_slot, n_slots <= 16; sorted by gid) and slot the
        LAST logged DECISION and ACCEPT image and the ring position of the accept's request blob.  -> [n, 16] log_hit."""
        wants = np.ascontiguousarray(wants, dtype=log_want_dtype)
        n = len(wants)
        out = np.zeros((max(n, 1), GPX_LOG_SPAN), dtype=log_hit_dtype)
        self.L.check(self.L.fn("log_find")(self._h, C.c_uint32(lane), C.c_uint64(from_), C.c_uint32(n), _ptr(wants), _ptr(out)))
        return out[:n]

    def select_groups(self, lane: int, mask: int, value: int, cap: Optional[int] = None) -> np.ndarray:
        """The live, ACTIVE groups of `lane` with (flag byte & mask) == value, ascending (gpx_select_groups): the slow-path
        list (mask = value = GF_NEEDS_SYNC) or the pause candidates (mask = GF_NOT_CAUGHT_UP, value = 0)."""
        cap = int(self.cfg.max_groups) if cap is None else int(cap)
        out = np.zeros(max(cap, 1), dtype=np.uint32)
        n = C.c_uint32(0)
        self.L.check(self.L.fn("select_groups")(self._h, C.c_uint32(lane), C.c_uint32(mask), C.c_uint32(value), _ptr(out),
                                                C.c_uint32(cap), C.byref(n)))
        if n.value > cap:
            raise GpxError(GPX_ERANGE, f"{n.value} groups match, buffer holds {cap}")
        return out[: n.value].copy()

    def missing_decisions(self, lane: int, gids, size_limit: int = 400, too_much_gap: int = 400) -> np.ndarray:
        """The fields of a SYNC_DECISIONS_REQUEST per group (gpx_missing_decisions): PISM.requestMissingDecisions :2292."""
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        out = np.zeros(max(len(gids), 1), dtype=missing_dtype)
        self.L.check(self.L.fn("missing_decisions")(self._h, C.c_uint32(lane), C.c_uint32(len(gids)), _ptr(gids),
                                                    C.c_int32(size_limit), C.c_int32(too_much_gap), _ptr(out)))
        return out[: len(gids)]

    def clear_group_flags(self, lane: int, gids, mask: int):
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        self.L.check(self.L.fn("clear_group_flags")(self._h, C.c_uint32(lane), C.c_uint32(len(gids)), _ptr(gids), C.c_uint32(mask)))

    def log_gather(self, lane: int, positions, lengths) -> list:
        """The byte ranges [pos, pos + len) of `lane`'s log ring (request bodies of gpx_log_find hits / carried-over
        pvalues) in one call and one device->host copy (gpx_log_gather).  -> list of bytes."""
        n = len(positions)
        if n == 0:
            return []
        r = np.zeros(n, dtype=log_range_dtype)
        r["pos"], r["len"] = positions, lengths
        padded = (r["len"].astype(np.uint64) + 15) // 16 * 16
        offs = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.uint64)
        r["dst_off"] = offs
        total = int(padded.sum())
        buf = np.zeros(max(total, 16), dtype=np.uint8)
        self.L.check(self.L.fn("log_gather")(self._h, C.c_uint32(lane), C.c_uint32(n), _ptr(r), _ptr(buf), C.c_uint64(total)))
        return [bytes(buf[int(o): int(o) + int(l)]) for o, l in zip(offs, r["len"])]

    def pause_groups(self, gids):
        """The deactivation sweep (gpx_pause_groups): -> (rows [n, n_lanes] of gpx_row, paused [n] bool).  Rows of groups
        that did not pause are zero."""
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        n = len(gids)
        rows = np.zeros((max(n, 1), self.n_lanes), dtype=row_dtype)
        paused = np.zeros(max(n, 1), dtype=np.uint8)
        self.L.check(self.L.fn("pause_groups")(self._h, C.c_uint32(n), _ptr(gids), _ptr(rows), _ptr(paused)))
        return rows[:n], paused[:n].astype(bool)

    def patch(self, patches: np.ndarray):
        patches = np.ascontiguousarray(patches, dtype=patch_dtype)
        self.L.check(self.L.fn("patch")(self._h, C.c_uint32(len(patches)), _ptr(patches)))

    def group_flags(self, gids, lane: int) -> np.ndarray:
        gids = np.ascontiguousarray(gids, dtype=np.uint32)
        out = np.zeros(len(gids), dtype=np.uint8)
        self.L.check(self.L.fn("get_group_flags")(self._h, C.c_uint32(lane), C.c_uint32(len(gids)), _ptr(gids),
                                                  _ptr(out)))
        return out

    # ---- response cache: device buffers (torch CUDA tensors), on `stream` (None: torch's current stream) ----------
    def response_cache_init(self, n_buckets: int, timeout_ms: int):
        """gpx_response_cache_init: an empty table of n_buckets buckets whose entries expire after timeout_ms"""
        self.L.check(self.L.fn("response_cache_init")(self._h, C.c_uint32(n_buckets), C.c_int64(timeout_ms)))

    def response_cache_put(self, keys, n: int, now_ms: int, stream=None):
        """gpx_response_cache_put_device: the first n rows of keys (rc_key_dtype records, [k, 24] uint8) at now_ms"""
        from .wire import _dptr, stream_handle
        self.L.check(self.L.fn("response_cache_put_device")(self._h, C.c_uint32(n), _dptr(keys), C.c_int64(now_ms),
                                                             stream_handle(stream)))

    def response_cache_match(self, reqs, meta, n: int, now_ms: int, hit, out_reqs, out_meta, stream=None) -> int:
        """gpx_response_cache_match_device over the first n rows of reqs / meta ([k, 32] uint8, a request decoder's
        output): hit int32 [n] receives each request's handle or -1, out_reqs / out_meta the misses in input order.
        -> the count of misses"""
        from .wire import _dptr, stream_handle
        n_out = C.c_uint32(0)
        self.L.check(self.L.fn("response_cache_match_device")(self._h, C.c_uint32(n), _dptr(reqs), _dptr(meta),
                                                               C.c_int64(now_ms), _dptr(hit), _dptr(out_reqs),
                                                               _dptr(out_meta), C.byref(n_out),
                                                               stream_handle(stream)))
        return n_out.value

    # ---- data path ------------------------------------------------------------------
    def propose(self, reqs: np.ndarray, payload: np.ndarray):
        reqs = np.ascontiguousarray(reqs, dtype=request_dtype)
        payload = np.ascontiguousarray(payload, dtype=np.uint8)
        n = len(reqs)
        pal = (payload.size + 15) & ~15
        accepts = np.zeros(max(n, 1), dtype=accept_dtype)
        blob = np.zeros(2 * pal + 16 * n + 64, dtype=np.uint8)
        status = np.zeros(max(n, 1), dtype=np.int32)
        na, bb = C.c_uint32(0), C.c_uint64(0)
        self.L.check(self.L.fn("propose")(self._h, C.c_uint32(n), _ptr(reqs), _ptr(payload),
                                          C.c_uint64(payload.size), _ptr(accepts), C.byref(na), _ptr(blob),
                                          C.c_uint64(blob.size), C.byref(bb), _ptr(status)))
        return accepts[: na.value].copy(), blob[: bb.value].copy(), status[:n].copy()

    def handle_accepts(self, accepts: np.ndarray, blob: np.ndarray, extra_cap: int = 4096):
        accepts = np.ascontiguousarray(accepts, dtype=accept_dtype)
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        if blob.size & 15:
            blob = np.concatenate([blob, np.zeros(16 - (blob.size & 15), dtype=np.uint8)])
        n = len(accepts)
        replies = np.zeros(max(n * self.n_lanes, 1), dtype=reply_dtype)
        extra = np.zeros(max(extra_cap, 1), dtype=exec_dtype)
        nx = C.c_uint32(0)
        self.L.check(self.L.fn("handle_accepts")(self._h, C.c_uint32(n), _ptr(accepts), _ptr(blob),
                                                 C.c_uint64(blob.size), _ptr(replies), _ptr(extra),
                                                 C.c_uint32(extra_cap), C.byref(nx)))
        return replies[: n * self.n_lanes].copy(), extra[: min(nx.value, extra_cap)].copy()

    def handle_accept_replies(self, replies: np.ndarray) -> np.ndarray:
        replies = np.ascontiguousarray(replies, dtype=reply_dtype)
        n = len(replies)
        dec = np.zeros(max(n, 1), dtype=decision_dtype)
        nd = C.c_uint32(0)
        self.L.check(self.L.fn("handle_accept_replies")(self._h, C.c_uint32(n), _ptr(replies), _ptr(dec),
                                                        C.byref(nd)))
        return dec[: nd.value].copy()

    def handle_decisions(self, decisions: np.ndarray, extra_cap: int = 4096):
        decisions = np.ascontiguousarray(decisions, dtype=decision_dtype)
        n = len(decisions)
        ex = np.zeros(max(n * self.n_lanes, 1), dtype=exec_dtype)
        extra = np.zeros(max(extra_cap, 1), dtype=exec_dtype)
        nx = C.c_uint32(0)
        self.L.check(self.L.fn("handle_decisions")(self._h, C.c_uint32(n), _ptr(decisions), _ptr(ex), _ptr(extra),
                                                   C.c_uint32(extra_cap), C.byref(nx)))
        return ex[: n * self.n_lanes].copy(), extra[: min(nx.value, extra_cap)].copy()

    def handle_prepares(self, prepares: np.ndarray) -> np.ndarray:
        """PISM.handlePrepare at every addressed local lane; `prepares` are pvalue headers (slot = firstUndecidedSlot).
        Returns prepare_reply records, shape [n * n_lanes]."""
        prepares = np.ascontiguousarray(prepares, dtype=decision_dtype)
        n = len(prepares)
        out = np.zeros(max(n * self.n_lanes, 1), dtype=prepare_reply_dtype)
        self.L.check(self.L.fn("handle_prepares")(self._h, C.c_uint32(n), _ptr(prepares), _ptr(out)))
        return out[: n * self.n_lanes]

    def handle_prepare_replies(self, elections: np.ndarray, replies: np.ndarray) -> np.ndarray:
        """Phase 1b for a batch of elections (PISM.handlePrepareReply :1017-1068 and what follows a majority:
        carry-over, no-op fill, processStop, the coordinator installed ACTIVE).  Returns election_out records."""
        elections = np.ascontiguousarray(elections, dtype=election_dtype)
        replies = np.ascontiguousarray(replies, dtype=prepare_reply_dtype)
        n = len(elections)
        out = np.zeros(max(n, 1), dtype=election_out_dtype)
        self.L.check(self.L.fn("handle_prepare_replies")(self._h, C.c_uint32(n), _ptr(elections), C.c_uint32(len(replies)),
                                                         _ptr(replies), _ptr(out)))
        return out[:n]

    def handle_accepts_fused(self, accepts: np.ndarray, blob: np.ndarray, extra_cap: int = 4096):
        accepts = np.ascontiguousarray(accepts, dtype=accept_dtype)
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        if blob.size & 15:
            blob = np.concatenate([blob, np.zeros(16 - (blob.size & 15), dtype=np.uint8)])
        n = len(accepts)
        replies = np.zeros(max(n * self.n_lanes, 1), dtype=reply_dtype)
        dec = np.zeros(max(n, 1), dtype=decision_dtype)
        ex = np.zeros(max(n * self.n_lanes, 1), dtype=exec_dtype)
        extra = np.zeros(max(extra_cap, 1), dtype=exec_dtype)
        nx = C.c_uint32(0)
        self.L.check(self.L.fn("handle_accepts_fused")(self._h, C.c_uint32(n), _ptr(accepts), _ptr(blob),
                                                       C.c_uint64(blob.size), _ptr(replies), _ptr(dec), _ptr(ex),
                                                       _ptr(extra), C.c_uint32(extra_cap), C.byref(nx)))
        return (replies[: n * self.n_lanes].copy(), dec[:n].copy(), ex[: n * self.n_lanes].copy(),
                extra[: min(nx.value, extra_cap)].copy())

    def round_phases(self, reqs: np.ndarray, payload: np.ndarray, extra_cap: int = 4096):
        return self.round(reqs, payload, extra_cap, fn="round_phases")

    def round(self, reqs: np.ndarray, payload: np.ndarray, extra_cap: int = 4096, fn: str = "round"):
        reqs = np.ascontiguousarray(reqs, dtype=request_dtype)
        payload = np.ascontiguousarray(payload, dtype=np.uint8)
        n = len(reqs)
        status = np.zeros(max(n, 1), dtype=np.int32)
        ex = np.zeros(max(n * self.n_lanes, 1), dtype=exec_dtype)
        extra = np.zeros(max(extra_cap, 1), dtype=exec_dtype)
        ns, nx = C.c_uint32(0), C.c_uint32(0)
        self.L.check(self.L.fn(fn)(self._h, C.c_uint32(n), _ptr(reqs), _ptr(payload), C.c_uint64(payload.size),
                                        _ptr(status), _ptr(ex), C.byref(ns), _ptr(extra), C.c_uint32(extra_cap),
                                        C.byref(nx)))
        return status[:n].copy(), ex[: ns.value].copy(), extra[: min(nx.value, extra_cap)].copy()

    # ---- pipelined rounds (gpx_round_submit / gpx_round_wait) ---------------------------
    def round_submit(self, reqs: np.ndarray, payload: np.ndarray, compact: bool = False, extra_cap: int = 4096,
                     bufs: Optional[dict] = None, packed: bool = False) -> int:
        """Enqueue one round; returns its ticket.  `bufs` may carry caller-owned (e.g. page-locked) output arrays
        `status`, `exec`, `sum`, `extra`; otherwise they are allocated here and returned by round_wait."""
        assert reqs.dtype == (request_packed_dtype if packed else request_dtype)
        assert reqs.flags.c_contiguous and payload.dtype == np.uint8
        n = len(reqs)
        b = dict(bufs or {})
        if compact:
            b.setdefault("sum", np.zeros(max(n, 1), dtype=exec_sum_dtype))
        else:
            b.setdefault("status", np.zeros(max(n, 1), dtype=np.int32))
            b.setdefault("exec", np.zeros(max(n * self.n_lanes, 1), dtype=exec_dtype))
        b.setdefault("extra", np.zeros(max(extra_cap, 1), dtype=exec_dtype))
        io = RoundIO(n, (ROUND_COMPACT if compact else 0) | (ROUND_PACKED_REQS if packed else 0), reqs.ctypes.data, payload.ctypes.data if payload.size else None,
                     payload.size, b["status"].ctypes.data if "status" in b else None,
                     b["exec"].ctypes.data if "exec" in b else None, b["sum"].ctypes.data if "sum" in b else None,
                     b["extra"].ctypes.data, len(b["extra"]))
        t = C.c_uint64(0)
        self.L.check(self.L.fn("round_submit")(self._h, C.byref(io), C.byref(t)))
        b["n"], b["compact"], b["reqs"], b["payload"] = n, compact, reqs, payload  # keep the inputs alive
        self._inflight[t.value] = b
        return t.value

    def round_wait(self, ticket: int) -> dict:
        """Block until round `ticket` is done; returns {status, exec | sum, extra (trimmed), n_extra}."""
        ns, nx = C.c_uint32(0), C.c_uint32(0)
        self.L.check(self.L.fn("round_wait")(self._h, C.c_uint64(ticket), C.byref(ns), C.byref(nx)))
        b = self._inflight.pop(ticket)
        n = b["n"]
        out = {"n_extra": nx.value, "extra": b["extra"][: min(nx.value, len(b["extra"]))]}
        if b["compact"]:
            out["sum"] = b["sum"][:n]
        else:
            out["status"], out["exec"] = b["status"][:n], b["exec"][: ns.value]
        return out

    def digest_requests(self, reqs: np.ndarray, payload: np.ndarray) -> np.ndarray:
        """MD5 of every requestValue (RequestPacket.getDigest), shape [n, 16]."""
        reqs = np.ascontiguousarray(reqs, dtype=request_dtype)
        payload = np.ascontiguousarray(payload, dtype=np.uint8)
        out = np.zeros((max(len(reqs), 1), 16), dtype=np.uint8)
        self.L.check(self.L.fn("digest_requests")(self._h, C.c_uint32(len(reqs)), _ptr(reqs), _ptr(payload),
                                                  C.c_uint64(payload.size), _ptr(out)))
        return out[: len(reqs)]

    # ---- log / counters --------------------------------------------------------------
    def log_head(self, lane: int) -> int:
        head = C.c_uint64(0)
        self.L.check(self.L.fn("log_read")(self._h, C.c_uint32(lane), C.c_uint64(0), None, C.c_uint64(0), None,
                                           C.byref(head)))
        return head.value

    def log_read(self, lane: int, start: int = 0, nbytes: Optional[int] = None) -> np.ndarray:
        head = self.log_head(lane)
        if nbytes is None:
            nbytes = max(head - start, 0)
        buf = np.zeros(max(nbytes, 1), dtype=np.uint8)
        got = C.c_uint64(0)
        self.L.check(self.L.fn("log_read")(self._h, C.c_uint32(lane), C.c_uint64(start), _ptr(buf),
                                           C.c_uint64(nbytes), C.byref(got), None))
        return buf[: got.value]

    def log_drain_async(self, lane: int, dst_ptr: int, cap: int, after_stream: int = 0):
        """enqueue the copy of the next undrained ring bytes into host memory at dst_ptr; returns (from, n_bytes)"""
        f, nb = C.c_uint64(0), C.c_uint64(0)
        self.L.check(self.L.fn("log_drain_async")(self._h, C.c_uint32(lane), C.c_void_p(dst_ptr), C.c_uint64(cap),
                                                  C.byref(f), C.byref(nb), C.c_void_p(after_stream) if after_stream else None))
        return f.value, nb.value

    def log_frame_device(self, lane: int, from_: int, meta, n_meta: int, caps=(0, 0, 0), stream=None):
        """gpx_log_frame_device: the journal frames of [from_, head) of `lane`'s ring.  meta: a CUDA tensor of n_meta
        journal_req_dtype records ([n, 24] uint8, ascending by (gid, req_id)), or None.  caps = (frame bytes, frames,
        misses); on GPX_ERANGE the outputs are allocated again at the sizes the call reports and the call is repeated.
        -> LogFrames(rc, the new from, frames uint8 [bytes], missing [k, 16] (journal_miss_dtype rows), sizes); rc is
        GPX_OK or GPX_ENOENT (no frame written, from unchanged), any other code raises."""
        import torch
        from .wire import _dptr, _on, stream_handle
        dev = meta.device if meta is not None else torch.device("cuda", torch.cuda.current_device())
        caps = [int(c) for c in caps]
        with _on(stream):
            for _ in range(2):
                out = torch.empty(max(caps[0], 1), dtype=torch.uint8, device=dev)
                miss = torch.empty((max(caps[2], 1), 16), dtype=torch.uint8, device=dev)
                f, ob, nf, nm = C.c_uint64(from_), C.c_uint64(caps[0]), C.c_uint32(caps[1]), C.c_uint32(caps[2])
                rc = self.L.fn("log_frame_device")(self._h, C.c_uint32(lane), C.byref(f), _dptr(meta),
                                                   C.c_uint32(n_meta), _dptr(out), C.byref(ob), C.byref(nf),
                                                   _dptr(miss), C.byref(nm), stream_handle(stream))
                caps = [ob.value, nf.value, nm.value]
                if rc != GPX_ERANGE:
                    break
        if rc not in (GPX_OK, GPX_ENOENT):
            self.L.check(rc)
        return LogFrames(rc, f.value, out[: caps[0]], miss[: caps[2]], tuple(caps))

    def journal_compact_device(self, data, n_bytes: int, file_off, starts, gc_slot, last_readonly: bool,
                               caps=(0, 0), stream=None):
        """gpx_journal_compact_device over CUDA tensors: data (uint8, the files concatenated), file_off (uint32 [k+1]),
        starts (uint32 frame offsets), gc_slot (int32 per gid).  caps = (out bytes, bad frames); on GPX_ERANGE the
        outputs are allocated again at the sizes the call reports and the call is repeated.  -> JournalCompact(rc, out
        uint8 [bytes], files [k, 24] (journal_file_dtype rows), bad uint32 frame indices, sizes); rc is GPX_OK or
        GPX_EINVAL with bad listed (nothing else written), any other code raises."""
        import torch
        from .wire import _dptr, _on, stream_handle
        k = int(file_off.numel()) - 1
        caps = [int(c) for c in caps]
        with _on(stream):
            for _ in range(2):
                out = torch.empty(max(caps[0], 1), dtype=torch.uint8, device=data.device)
                files = torch.empty((max(k, 1), 24), dtype=torch.uint8, device=data.device)
                bad = torch.empty(max(caps[1], 1), dtype=torch.int32, device=data.device)
                ob, nb = C.c_uint64(caps[0]), C.c_uint32(caps[1])
                rc = self.L.fn("journal_compact_device")(
                    self._h, _dptr(data), C.c_uint64(n_bytes), _dptr(file_off), C.c_uint32(k), _dptr(starts),
                    C.c_uint32(int(starts.numel())), _dptr(gc_slot), C.c_uint32(int(gc_slot.numel())),
                    C.c_uint32(1 if last_readonly else 0), _dptr(out), C.byref(ob), _dptr(files), _dptr(bad),
                    C.byref(nb), stream_handle(stream))
                caps = [ob.value, nb.value]
                if rc != GPX_ERANGE:
                    break
        if rc == GPX_EINVAL and caps[1]:
            return JournalCompact(rc, out[:0], files[:0], bad[: caps[1]], tuple(caps))
        self.L.check(rc)
        return JournalCompact(rc, out[: caps[0]], files[:k], bad[:0], tuple(caps))

    def log_drain_wait(self):
        self.L.check(self.L.fn("log_drain_wait")(self._h))

    def log_release(self, lane: int, upto: int):
        self.L.check(self.L.fn("log_release")(self._h, C.c_uint32(lane), C.c_uint64(upto)))

    def counters(self) -> dict:
        c = Counters()
        self.L.check(self.L.fn("get_counters")(self._h, C.byref(c)))
        return {n: int(getattr(c, n)) for n in COUNTER_NAMES}

    def reset_counters(self):
        self.L.check(self.L.fn("reset_counters")(self._h))


def seg_end(off: int, hdr) -> int:
    """Where the segment whose header `hdr` sits at ring offset `off` ends (seg_end in gpx_dev.cuh)."""
    return (off + 64 + int(hdr["n_slots"]) * int(hdr["rec_bytes"]) + ((int(hdr["payload_bytes"]) + 15) & ~15)
            + 31) & ~31


def parse_log(buf: np.ndarray, ring_cap: Optional[int] = None, base: int = 0):
    """Walk the segments of a log ring image.  Returns [(hdr, images, payload_area, payload_ring_off)].

    Without ring_cap the walk stops at the first header whose magic does not match.  With ring_cap, buf holds a
    device ring's bytes from the absolute ring offset `base` on, and a segment counts only when its magic matches and
    its ring_off is base + its offset in buf (the rule k_log_dir applies).  Anything else is the tail a launch skipped
    because it would have straddled the ring end, and may hold stale segments of an earlier lap: the walk goes on at
    the next lap."""
    out = []
    off = 0
    n = buf.size
    while off + 64 <= n:
        hdr = buf[off: off + 64].view(seg_hdr_dtype)[0]
        if int(hdr["magic"]) != SEG_MAGIC or (ring_cap and int(hdr["ring_off"]) != base + off):
            if not ring_cap:
                break
            nxt = ((base + off) // ring_cap + 1) * ring_cap - base
            if nxt <= off or nxt + 64 > n:
                break
            off = nxt
            continue
        rec = int(hdr["rec_bytes"])
        ns = int(hdr["n_slots"])
        nv = int(hdr["n_valid"])
        pb = int(hdr["payload_bytes"])
        if rec == 48:  # two planes: ns x 32 B pvalue headers, then ns x 16 B extensions
            imgs = np.zeros(nv, dtype=accept_dtype)
            hp = buf[off + 64: off + 64 + ns * 32].view(decision_dtype)[:nv]
            xp = buf[off + 64 + ns * 32: off + 64 + ns * 48].view(
                np.dtype([("payload_off", "<u4"), ("payload_len", "<u4"), ("nreq", "<u4"), ("sender", "<i4")]))[:nv]
            for f in decision_dtype.names:
                imgs[f] = hp[f]
            for f in xp.dtype.names:
                imgs[f] = xp[f]
        else:
            imgs = buf[off + 64: off + 64 + ns * rec].view(decision_dtype)[:nv]
        pay_off = off + 64 + ns * rec
        payload = buf[pay_off: pay_off + pb]
        out.append((hdr, imgs, payload, pay_off))
        off = seg_end(base + off, hdr) - base
    return out
