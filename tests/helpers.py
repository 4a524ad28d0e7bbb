"""Shared test helpers: library loading, synthetic workloads, output canonicalisation."""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from gigapaxos_b200 import abi  # noqa: E402
from gigapaxos_b200.abi import Engine, Library  # noqa: E402
from gigapaxos_b200.abi import GpxError as GpxErrorT  # noqa: E402

ORACLE_PATH = os.path.join(ROOT, "oracle", "libgpx_oracle.so")
_oracle = None
_emu = {}  # (source, defines) -> the emulated library (emu_libraries)


def oracle_library() -> Library:
    """The CPU oracle behind the same wrapper (tests only)."""
    global _oracle
    if _oracle is None:
        if not os.path.exists(ORACLE_PATH):
            from gigapaxos_b200 import build
            build.build_oracle()
        _oracle = Library(ORACLE_PATH, "gpxo_")
    return _oracle


def ptr(a):
    """a numpy array's data as a ctypes pointer; None stays a null pointer"""
    import ctypes as C
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def emu_libraries(tmp_path_factory, *sources, defines=()):
    """tests/emu/<source>.cpp for each source, kernel sources compiled for the host with the -D `defines` (under
    AddressSanitizer + UBSan when GPX_EMU_SANITIZE is set) -> {source: library}.  Each (source, defines) is built once
    per process, the missing ones at the same time; skips the test without the CUDA headers."""
    import ctypes as C
    import subprocess

    import pytest
    cuda_inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("no CUDA headers")
    sanitize = (["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-g"]
                if os.environ.get("GPX_EMU_SANITIZE") else [])
    defines = tuple(defines)
    jobs = []
    for src in sources:
        if (src, defines) not in _emu:
            out = str(tmp_path_factory.mktemp("emu") / f"lib{src}.so")
            jobs.append((src, out, subprocess.Popen(
                ["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", *sanitize, *(f"-D{d}" for d in defines),
                 "-I", cuda_inc, "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "gigapaxos_b200", "csrc"),
                 "-x", "c++", os.path.join(ROOT, "tests", "emu", src + ".cpp"), "-o", out])))
    for src, out, p in jobs:
        assert p.wait() == 0, f"g++ {src}.cpp"
        lib = _emu[(src, defines)] = C.CDLL(out)
        lib.emu_set_order.argtypes = [C.c_char_p]
        if hasattr(lib, "emu_last_error"):  # the libraries that run the engine's sequences
            lib.emu_last_error.restype = C.c_char_p
        if hasattr(lib, "emu_wire_new"):  # the wire libraries' world
            lib.emu_wire_new.restype = C.c_void_p
            lib.emu_wire_new.argtypes = [C.c_uint32, C.c_uint32, C.c_void_p]
    return {src: _emu[(src, defines)] for src in sources}


def emu_library(tmp_path_factory, source, *defines):
    """emu_libraries for one source"""
    return emu_libraries(tmp_path_factory, source, defines=defines)[source]


def make_config(lib: Library, **kw) -> abi.Config:
    cfg = lib.config_defaults()
    for k, v in kw.items():
        if k == "lane_node":
            for i, x in enumerate(v):
                cfg.lane_node[i] = int(x)
        else:
            setattr(cfg, k, v)
    return cfg


def splitmix64(x: np.ndarray) -> np.ndarray:
    x = (x + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
    z = x
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def group_names(n: int, prefix: str = "NoopPaxosApp") -> list[str]:
    return [f"{prefix}{i}" for i in range(n)]


def group_descs(n: int, members=(100, 101, 102), init_mode=abi.INIT_BATCH, prefix="NoopPaxosApp", gid0=0,
                version=0) -> np.ndarray:
    d = np.zeros(n, dtype=abi.group_desc_dtype)
    d["gid"] = np.arange(gid0, gid0 + n, dtype=np.uint32)
    d["version"] = version
    d["name_hash"] = [abi.java_string_hash(s) for s in group_names(n, prefix)]
    d["n_members"] = len(members)
    for i, m in enumerate(members):
        d["members"][:, i] = m
    d["init_mode"] = init_mode
    return d


def make_requests(gids, payload_len=1, seed=1, entry_lane=0, entry_node=100, stop_mask=None, round_no=0):
    """One request per entry of `gids` (already grouped by gid), payloads 16-B aligned in the arena."""
    gids = np.asarray(gids, dtype=np.uint32)
    n = len(gids)
    lens = np.broadcast_to(np.asarray(payload_len, dtype=np.uint32), (n,)).copy()
    stride = ((lens + 15) // 16) * 16
    offs = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint32) if n else np.zeros(0, np.uint32)
    total = int(stride.sum())
    rng = np.random.default_rng(seed + 7919 * round_no)
    alphabet = np.frombuffer(b"0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    payload = np.zeros(total, dtype=np.uint8)
    for i in range(n):
        payload[offs[i]: offs[i] + lens[i]] = alphabet[rng.integers(0, 62, size=int(lens[i]))]
    reqs = np.zeros(n, dtype=abi.request_dtype)
    reqs["gid"] = gids
    flags = np.full(n, (entry_lane & 0xF) << 8, dtype=np.uint32)
    if stop_mask is not None:
        flags |= np.where(np.asarray(stop_mask), abi.F_STOP, 0).astype(np.uint32)
    reqs["flags"] = flags
    idx = np.arange(n, dtype=np.uint64) + np.uint64(round_no) * np.uint64(1 << 32) + np.uint64(seed) * np.uint64(1 << 48)
    reqs["req_id"] = (splitmix64(idx) & np.uint64(0x7FFFFFFFFFFFFFFF)).astype(np.int64)
    reqs["payload_off"] = offs
    reqs["payload_len"] = lens
    reqs["entry_node"] = entry_node
    reqs["client"] = np.arange(n, dtype=np.uint32)
    return reqs, payload


def canon(recs: np.ndarray, keys=("gid",)) -> np.ndarray:
    """Stable-sort records by group (order inside a group is preserved) and drop VOID holes."""
    if len(recs) == 0:
        return recs
    names = recs.dtype.names
    if "who" in names:
        keep = (abi.who_flags(recs["who"]) & abi.F_VOID) == 0
    else:
        keep = (recs["flags"] & abi.F_VOID) == 0
    r = recs[keep]
    order = np.argsort(r["gid"], kind="stable")
    return r[order]


def exec_by_lane(ex: np.ndarray, n_lanes: int) -> list[np.ndarray]:
    lanes = (ex["flags"] >> 12) & 0xF
    out = []
    for l in range(n_lanes):
        e = ex[(lanes == l) & ((ex["flags"] & abi.F_VOID) == 0)]
        out.append(e[np.argsort(e["gid"], kind="stable")])
    return out


def java_hash_numbered(prefix: str, idx: np.ndarray) -> np.ndarray:
    """String.hashCode() of f"{prefix}{i}" for every i of `idx`, vectorised (10 M names in about a second)."""
    idx = np.asarray(idx, dtype=np.int64)
    h0 = np.uint32(abi.java_string_hash(prefix) & 0xFFFFFFFF)
    out = np.zeros(len(idx), dtype=np.uint32)
    ndig = np.ones(len(idx), dtype=np.int64)
    t = idx // 10
    while np.any(t > 0):
        ndig += (t > 0)
        t //= 10
    for nd in np.unique(ndig):
        sel = np.nonzero(ndig == nd)[0]
        v = idx[sel]
        h = np.full(len(sel), h0, dtype=np.uint32)
        for k in range(int(nd) - 1, -1, -1):
            digit = (v // (10 ** k)) % 10
            with np.errstate(over="ignore"):
                h = h * np.uint32(31) + (digit + 48).astype(np.uint32)
        out[sel] = h
    return out.view(np.int32)


def group_descs_fast(n: int, members=(100, 101, 102), init_mode=abi.INIT_BATCH, prefix="NoopPaxosApp", gid0=0,
                     name0=0) -> np.ndarray:
    """group_descs for millions of groups (vectorised name hashes): gids gid0.., names prefix<name0 + k>"""
    d = np.zeros(n, dtype=abi.group_desc_dtype)
    d["gid"] = np.arange(gid0, gid0 + n, dtype=np.uint32)
    d["name_hash"] = java_hash_numbered(prefix, np.arange(name0, name0 + n))
    d["n_members"] = len(members)
    for i, m in enumerate(members):
        d["members"][:, i] = m
    d["init_mode"] = init_mode
    return d


def make_requests_fast(gids, payload_len=1, seed=1, entry_lane=0, entry_node=100, round_no=0, stride=None):
    """make_requests without the per-request Python loop (fixed payload length): full-size parity runs"""
    gids = np.asarray(gids, dtype=np.uint32)
    n = len(gids)
    P = int(payload_len)
    stride = ((P + 15) // 16) * 16 if stride is None else int(stride)
    rng = np.random.default_rng(seed + 7919 * round_no)
    alphabet = np.frombuffer(b"0123456789ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz", dtype=np.uint8)
    pay = np.zeros((n, stride), dtype=np.uint8)
    pay[:, :P] = alphabet[rng.integers(0, 62, size=(n, P))]
    reqs = np.zeros(n, dtype=abi.request_dtype)
    reqs["gid"] = gids
    reqs["flags"] = (entry_lane & 0xF) << 8
    idx = np.arange(n, dtype=np.uint64) + np.uint64(round_no) * np.uint64(1 << 32) + np.uint64(seed) * np.uint64(1 << 48)
    reqs["req_id"] = (splitmix64(idx) & np.uint64(0x7FFFFFFFFFFFFFFF)).astype(np.int64)
    reqs["payload_off"] = np.arange(n, dtype=np.uint32) * np.uint32(stride)
    reqs["payload_len"] = P
    reqs["entry_node"] = entry_node
    reqs["client"] = np.arange(n, dtype=np.uint32)
    return reqs, pay.reshape(-1)


def relay_into_small_ring(buf, heads, cap):
    """lay the calls of an (unwrapped) oracle ring image into a ring of `cap` bytes the way the device does: a call that
    would straddle the ring end skips to the ring start (gpx_dev.cuh seg_base), later laps overwrite earlier ones, every
    segment header names its new absolute position.  -> (ring bytes, new head, {old segment offset: new position},
    [new position of every call])"""
    ring = np.zeros(cap, dtype=np.uint8)
    pos, seg_map, call_pos = 0, {}, []
    for b0, b1 in zip(heads[:-1], heads[1:]):
        n = b1 - b0
        assert n <= cap
        if (pos % cap) + n > cap:
            pos += cap - pos % cap
        call_pos.append(pos)
        chunk = buf[b0:b1].copy()
        off = 0
        while off + 64 <= n:  # re-stamp ring_off of every segment of the call
            hdr = chunk[off: off + 64].view(abi.seg_hdr_dtype)[0]
            assert int(hdr["magic"]) == abi.SEG_MAGIC and int(hdr["ring_off"]) == b0 + off
            seg_map[b0 + off] = pos + off
            chunk[off: off + 64].view(abi.seg_hdr_dtype)[0]["ring_off"] = pos + off
            off = abi.seg_end(off, hdr)
        assert off == n
        ring[pos % cap: pos % cap + n] = chunk
        pos += n
    return ring, pos, seg_map, call_pos
