"""CPU: gpx_log_frame_device's kernels (gigapaxos_b200/csrc/gpx_journal.cuh with k_log_dir) and its host sequence
(log_frame in gpx_wire_seq.h) compiled for the host (tests/emu/journal_emu.cpp), against journal.LogDrainer on the same
range of the same ring: the frames are byte-identical, at block sizes 1, 7 and 64.  The rings are the oracle engine's
(fused rounds, batched slots, partial ACCEPTs, a view change's PREPAREs), as they lie and re-laid into a small ring that
wraps, and segments laid out as the engine lays them where an edge is wanted: VOID holes, batched slots of up to 1,024
requests with mixed STOP bits, STOP decisions, int32 slot and ballot edges, int64 req_id and entry_time edges, names
that need escaping.  Misses, GPX_ERANGE, GPX_EINVAL, empty and overwritten ranges, and a round trip through
journal.read_journal / parse_packet.  Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from gigapaxos_b200 import journal
from helpers import ROOT, abi, emu_library, ptr, relay_into_small_ring
from test_log_find import logged_engine

BLOCKS = [1, 7, 64]
I32, I64 = (-(1 << 31), (1 << 31) - 1), (-(1 << 63), (1 << 63) - 1)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = emu_library(tmp_path_factory, "journal_emu")
    lib.emu_journal_new.restype = C.c_void_p
    lib.emu_journal_new.argtypes = [C.c_uint32, C.c_uint32]
    lib.emu_journal_free.argtypes = [C.c_void_p]
    lib.emu_journal_names.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emu_journal_names_remove.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    lib.emu_log_frame.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    return lib


def hard_names(G, rng):
    """paxosIDs that need escaping: quotes, backslashes, control bytes, 0x7f, bytes >= 0x80, up to GPX_WIRE_MAX_ID"""
    out = {}
    specials = b'"\\\x00\x01\x08\x09\x0a\x0c\x0d\x1f\x7f\x80\xa9\xe9\xff/ '
    for g in range(G):
        if g % 4 == 0:
            out[g] = b"NoopPaxosApp%d" % g
        else:
            n = int(rng.integers(1, 128)) if g % 4 != 3 else 127
            raw = bytes(rng.choice(np.frombuffer(specials + b"abcXYZ019", np.uint8), size=n))
            out[g] = (b"%d" % g + raw)[:127]
    return out


class Emu:
    """one lane's world in the emulator: the name table, then calls on ring images"""

    def __init__(self, lib, G, names, versions, lane=0):
        self.lib, self.h = lib, lib.emu_journal_new(G, lane)
        gids = np.array(sorted(names), np.uint32)
        staged = np.zeros((len(gids), 128), np.uint8)
        for k, g in enumerate(gids):
            staged[k, 0] = len(names[int(g)])
            staged[k, 1: 1 + len(names[int(g)])] = np.frombuffer(names[int(g)], np.uint8)
        ver = np.array([versions[int(g)] for g in gids], np.int32)
        lib.emu_journal_names(self.h, len(gids), ptr(gids), ptr(staged), ptr(ver))

    def close(self):
        self.lib.emu_journal_free(self.h)

    def frame(self, ring, cap, head, start, meta, block=64, caps=None):
        """-> (rc, from, frames, missing, sizes); sized first unless caps are given"""
        meta = np.ascontiguousarray(meta, abi.journal_req_dtype)
        f = np.array([start], np.uint64)

        def call(sz):
            out = np.full(max(int(sz[0]), 1), 0xCD, np.uint8)
            miss = np.zeros(max(int(sz[2]), 1), abi.journal_miss_dtype)
            miss.view(np.uint8)[:] = 0xCD
            f[0] = start
            rc = self.lib.emu_log_frame(self.h, ptr(ring), cap, head, ptr(f), ptr(meta) if len(meta) else None,
                                        len(meta), ptr(out), ptr(miss), ptr(sz), block)
            return rc, out, miss
        sz = np.array(caps if caps is not None else (0, 0, 0), np.uint64)
        rc, out, miss = call(sz)
        if caps is None and rc == abi.GPX_ERANGE:
            rc, out, miss = call(sz)
        return rc, int(f[0]), out, miss, tuple(int(x) for x in sz)


class RingView:
    """log_head / log_read of one lane over a ring image (positions modulo its size), for LogDrainer"""

    def __init__(self, ring, head, cap):
        class Cfg:
            log_ring_bytes = cap
        self.cfg, self.ring, self.head, self.cap = Cfg, ring, head, cap

    def log_head(self, lane):
        return self.head

    def log_read(self, lane, start, nbytes):
        return self.ring.take(np.arange(start, start + nbytes) % self.cap)


class Collect:
    """the Journaler side of LogDrainer, in memory"""

    def __init__(self):
        self.buf = bytearray()

    def append(self, packet):
        self.buf += struct.pack(">i", len(packet)) + packet

    def end_batch(self):
        pass


def table(meta):
    return {(int(m["gid"]), int(m["req_id"])): (int(m["entry_node"]), int(m["entry_time"])) for m in meta}


def log_drainer(ring, cap, head, start, names, versions, meta):
    t = table(meta)

    def lookup(gid, rid):
        name = names[gid].decode("iso-8859-1")
        if (gid, rid) not in t and rid == -1:  # LogDrainer's second lookup for a PREPARE: the name only
            return name, versions[gid], 0, 0
        node, et = t[(gid, rid)]
        return name, versions[gid], node, et
    d = journal.LogDrainer(RingView(ring, head, cap), 0, Collect(), lookup)
    d.offset = start
    d.drain()
    return bytes(d.j.buf), d


def images(ring, cap, head, start):
    """(image, blob bytes or None) of every image in [start, head), in log order (VOID ones included)"""
    buf = ring.take(np.arange(start, head) % cap) if head > start else np.zeros(0, np.uint8)
    out = []
    for hdr, imgs, payload, _ in abi.parse_log(buf, cap, start):
        for im in imgs:
            blob = None
            if int(hdr["rec_bytes"]) == 48:
                blob = payload[int(im["payload_off"]): int(im["payload_off"]) + int(im["payload_len"])].tobytes()
            out.append((int(hdr["rec_bytes"]), im, blob))
    return out


def requests_of(ring, cap, head, start):
    """every (gid, req_id) a frame of the range looks up"""
    keys = set()
    for rec, im, blob in images(ring, cap, head, start):
        fl = int(im["flags"])
        if fl & abi.F_VOID or (rec == 32 and fl & abi.F_PREPARE):
            continue
        keys.add((int(im["gid"]), int(im["req_id"])))
        if rec == 48 and int(im["nreq"]) > 1:
            for e in np.frombuffer(blob[: 16 * int(im["nreq"])], abi.batch_ent_dtype)[1:]:
                keys.add((int(im["gid"]), int(e["req_id"])))
    return keys


def make_meta(keys, rng):
    keys = sorted(keys)
    m = np.zeros(len(keys), abi.journal_req_dtype)
    if keys:
        m["gid"], m["req_id"] = np.array(keys, dtype=object).T
    m["entry_node"] = rng.choice([I32[0], I32[1], -1, 0, 100, 101, 102], size=len(keys))
    m["entry_time"] = rng.choice([I64[0], I64[1], -1, 0, 1760000000000, 1 << 40], size=len(keys))
    return m


def expected_misses(ring, cap, head, start, names, meta):
    t = table(meta)
    out = []
    for rec, im, blob in images(ring, cap, head, start):
        fl, gid = int(im["flags"]), int(im["gid"])
        if fl & abi.F_VOID:
            continue
        kind = abi.F_ACCEPT if rec == 48 else abi.F_PREPARE if fl & abi.F_PREPARE else abi.F_DECISION
        if gid not in names:
            out.append((gid, kind, -1))
            continue
        if kind == abi.F_PREPARE:
            continue
        if (gid, int(im["req_id"])) not in t:
            out.append((gid, kind, int(im["req_id"])))
        if rec == 48 and int(im["nreq"]) > 1:
            for e in np.frombuffer(blob[: 16 * int(im["nreq"])], abi.batch_ent_dtype)[1:]:
                if (gid, int(e["req_id"])) not in t:
                    out.append((gid, kind, int(e["req_id"])))
    return out


def check_same(emu, ring, cap, head, start, names, versions, meta, block):
    rc, f, out, _, sz = emu.frame(ring, cap, head, start, meta, block)
    want, d = log_drainer(ring, cap, head, start, names, versions, meta)
    assert rc == 0, rc
    assert f == head
    got = bytes(out[: sz[0]])
    assert got == want
    assert sz[1] == d.accepts_written + d.decisions_written
    assert all(b == 0xCD for b in out[sz[0]:])
    return got


def parse_frames(data):
    pkts, p = [], 0
    while p < len(data):
        (n,) = struct.unpack(">i", data[p: p + 4])
        pkts.append(data[p + 4: p + 4 + n])
        p += 4 + n
    return pkts


# ---- the oracle engine's rings ----------------------------------------------------------------------------------------
def oracle_ring(eng, lane):
    head = eng.log_head(lane)
    cap = 1 << int(np.ceil(np.log2(head + 64)))
    ring = np.zeros(cap, np.uint8)
    ring[:head] = eng.log_read(lane)
    return ring, cap, head


@pytest.mark.parametrize("block", BLOCKS)
def test_oracle_rings_frame_as_log_drainer_does(oracle_lib, lib, block, tmp_path):
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed=block)
    rng = np.random.default_rng(block)
    names = hard_names(G, rng)
    versions = {g: int(rng.choice([0, 1, I32[0], I32[1]])) for g in range(G)}
    emu = Emu(lib, G, names, versions)
    n_frames = 0
    for lane in range(3):
        ring, cap, head = oracle_ring(eng, lane)
        for start in (0, heads[lane][len(heads[lane]) // 2], head):
            meta = make_meta(requests_of(ring, cap, head, start), rng)
            got = check_same(emu, ring, cap, head, start, names, versions, meta, block)
            n_frames += len(parse_frames(got))
        # a round trip: the journal reader gets the images' fields back, image by image
        meta = make_meta(requests_of(ring, cap, head, 0), rng)
        rc, _, out, _, sz = emu.frame(ring, cap, head, 0, meta, block)
        path = tmp_path / f"log.{lane}"
        path.write_bytes(bytes(out[: sz[0]]))
        pkts = list(journal.read_journal(str(path)))
        live = [(rec, im, blob) for rec, im, blob in images(ring, cap, head, 0) if not int(im["flags"]) & abi.F_VOID]
        assert len(pkts) == len(live) == sz[1]
        t = table(meta)
        for pkt, (rec, im, blob) in zip(pkts, live):
            v = journal.parse_packet(pkt)
            gid = int(im["gid"])
            assert v["paxos_id"] == names[gid].decode("iso-8859-1") and v["version"] == versions[gid]
            assert (v["bnum"], v["bcoord"]) == (int(im["bnum"]), int(im["bcoord"]))
            if rec == 48:
                assert v["kind"] == "ACCEPT" and v["slot"] == int(im["slot"]) and v["sender"] == int(im["sender"])
                assert v["n_batched"] == max(int(im["nreq"]) - 1, 0)
                if int(im["nreq"]) <= 1:
                    assert v["value"] == blob and v["request_id"] == int(im["req_id"])
            elif int(im["flags"]) & abi.F_PREPARE:
                assert v["kind"] == "PREPARE" and v["first_undecided_slot"] == int(im["slot"])
            else:
                assert v["kind"] == "DECISION" and v["slot"] == int(im["slot"]) and v["request_id"] == int(im["req_id"])
                assert (v["entry_replica"], v["entry_time"]) == t[(gid, int(im["req_id"]))]
                assert v["stop"] == bool(int(im["flags"]) & abi.F_STOP)
    assert n_frames > 500
    emu.close()
    eng.close()


@pytest.mark.parametrize("block", BLOCKS)
def test_a_ring_that_wraps(oracle_lib, lib, block):
    """re-laid into a small ring: a range that starts mid-ring, one that crosses the wrap and a skipped tail, drains
    call by call that add up to one drain, and a start whose bytes are gone"""
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed=10 + block, rounds=9)
    rng = np.random.default_rng(block)
    names = {g: b"NoopPaxosApp%d" % g for g in range(G)}
    versions = {g: 0 for g in range(G)}
    emu = Emu(lib, G, names, versions)
    crossed = 0
    for lane in range(3):
        buf, hs = eng.log_read(lane), heads[lane]
        cap = 1 << int(np.ceil(np.log2(2.2 * max(b - a for a, b in zip(hs[:-1], hs[1:])))))
        ring, head, _, call_pos = relay_into_small_ring(buf, hs, cap)
        assert head > 2 * cap
        first = next(i for i, p in enumerate(call_pos) if head - p <= cap)
        meta = make_meta(requests_of(ring, cap, head, call_pos[first]), rng)
        whole = check_same(emu, ring, cap, head, call_pos[first], names, versions, meta, block)
        parts = b""
        ends = call_pos[first + 1:] + [head]
        for a, b in zip(call_pos[first:], ends):
            rc, f, out, _, sz = emu.frame(ring, cap, b, a, meta, block)
            assert rc == 0 and f == b
            parts += bytes(out[: sz[0]])
        assert parts == whole
        for a, b in zip(call_pos[first:], ends[1:]):  # two calls: some cross the ring end, over a skipped tail
            check_same(emu, ring, cap, b, a, names, versions, meta, block)
            crossed += int(a // cap != (b - 1) // cap)
        rc, f, out, _, _ = emu.frame(ring, cap, head, call_pos[0], meta, block)
        assert rc == abi.GPX_ERANGE and f == call_pos[0] and np.all(out == 0xCD)
    assert crossed > 0
    emu.close()
    eng.close()


# ---- segments laid out as the engine lays them, for the edges ------------------------------------------------------------
def seg_hdr(pos, typ, n, rec, pay=0):
    h = np.zeros(1, abi.seg_hdr_dtype)
    h["magic"], h["type"], h["n_slots"], h["n_valid"] = abi.SEG_MAGIC, typ, n, n
    h["payload_bytes"], h["ring_off"], h["rec_bytes"] = pay, pos, rec
    return h.view(np.uint8)


def acc_segment(pos, accs):
    """an ACCEPT segment at ring position pos: accs = [(pvalue fields, sender, [(req_id, stop, value)])]"""
    n = len(accs)
    hp = np.zeros(n, abi.decision_dtype)
    xp = np.zeros(n, np.dtype([("payload_off", "<u4"), ("payload_len", "<u4"), ("nreq", "<u4"), ("sender", "<i4")]))
    pay = bytearray()
    for i, (pv, sender, reqs) in enumerate(accs):
        for k, v in pv.items():
            hp[i][k] = v
        if len(reqs) == 1:
            blob = reqs[0][2]
        else:
            ents = np.zeros(len(reqs), abi.batch_ent_dtype)
            ents["req_id"] = [r[0] for r in reqs]
            ents["len"] = [len(r[2]) for r in reqs]
            ents["flags"] = [abi.F_STOP if r[1] else 0 for r in reqs]
            blob = ents.tobytes() + b"".join(r[2] for r in reqs)
        xp[i] = (len(pay), len(blob), len(reqs), sender)
        pay += blob + b"\0" * (-len(blob) % 16)
    body = hp.tobytes() + xp.tobytes() + bytes(pay)
    seg = seg_hdr(pos, abi.F_ACCEPT, n, 48, len(pay)).tobytes() + body
    return seg + b"\0" * (-len(seg) % 32)


def dec_segment(pos, decs, typ=abi.F_DECISION):
    d = np.zeros(len(decs), abi.decision_dtype)
    for i, pv in enumerate(decs):
        for k, v in pv.items():
            d[i][k] = v
    return seg_hdr(pos, typ, len(decs), 32).tobytes() + d.tobytes()


def edge_ring(rng, G):
    """ACCEPTs with batches of up to 1,024 requests and mixed STOP bits, VOID holes, slots -7..1 and the int32 edges,
    int64 req_id edges, STOP decisions and a PREPARE segment"""
    segs, pos = [], 0
    rid = iter(list(I64) + [-1, 0, 1] + [int(x) for x in rng.integers(-(1 << 62), 1 << 62, size=8000)])
    slots = list(range(-7, 2)) + [I32[0], I32[1], I32[1] - 1]
    ballots = [(0, 100), (I32[1], I32[0]), (I32[0], I32[1]), (-1, 101), (7, -5)]
    for s in range(3):
        accs = []
        for i, slot in enumerate(slots):
            nreq = [1, 2, 1024, 3, 1, 17][(i + s) % 6]
            reqs = [(next(rid), bool(rng.random() < 0.3), bytes(rng.integers(0, 256, size=int(rng.integers(0, 40)), dtype=np.uint8)))
                    for _ in range(nreq)]
            bn, bc = ballots[(i + s) % len(ballots)]
            flags = abi.F_ACCEPT | (abi.F_STOP if any(r[1] for r in reqs) else 0) | (abi.F_VOID if i % 5 == 4 else 0)
            pv = dict(gid=(i * 7 + s) % G, slot=slot, bnum=bn, bcoord=bc, median_cp=slots[-1 - i], flags=flags,
                      req_id=reqs[0][0])
            accs.append((pv, [I32[0], I32[1], 100, -1][i % 4], reqs))
        seg = acc_segment(pos, accs)
        segs.append(seg)
        pos += len(seg)
        decs = []
        for i, (pv, _, reqs) in enumerate(accs):
            decs.append(dict(pv, flags=abi.F_DECISION | abi.F_META | (abi.F_STOP if i % 3 == 0 else 0)
                             | (abi.F_VOID if i % 4 == 1 else 0), median_cp=-1))
        seg = dec_segment(pos, decs)
        segs.append(seg)
        pos += len(seg)
        preps = [dict(gid=g, slot=slots[g % len(slots)], bnum=ballots[g % 5][0], bcoord=ballots[g % 5][1],
                      flags=abi.F_PREPARE | (abi.F_VOID if g == 3 else 0), req_id=-1) for g in range(0, G, 3)]
        seg = dec_segment(pos, preps, abi.F_PREPARE)
        segs.append(seg)
        pos += len(seg)
    data = b"".join(segs)
    cap = 1 << int(np.ceil(np.log2(len(data) + 64)))
    ring = np.zeros(cap, np.uint8)
    ring[: len(data)] = np.frombuffer(data, np.uint8)
    return ring, cap, len(data), [sum(len(x) for x in segs[:k]) for k in range(len(segs) + 1)]


@pytest.mark.parametrize("block", BLOCKS)
def test_edges(lib, block):
    G = 24
    rng = np.random.default_rng(100 + block)
    ring, cap, head, bounds = edge_ring(rng, G)
    names = hard_names(G, rng)
    versions = {g: int(rng.choice([0, 3, I32[0], I32[1]])) for g in range(G)}
    emu = Emu(lib, G, names, versions)
    meta = make_meta(requests_of(ring, cap, head, 0), rng)
    got = check_same(emu, ring, cap, head, 0, names, versions, meta, block)
    for start in bounds[1:-1:2]:
        check_same(emu, ring, cap, head, start, names, versions, meta, block)
    kinds = [journal.parse_packet(p)["kind"] for p in parse_frames(got)]
    assert {"ACCEPT", "DECISION", "PREPARE"} == set(kinds)
    v = [journal.parse_packet(p) for p in parse_frames(got)]
    assert max(x["n_batched"] for x in v if x["kind"] == "ACCEPT") == 1023
    assert any(x["stop"] for x in v if x["kind"] == "DECISION") and {I32[1], -7, 0, 1} <= {x["slot"] for x in v if "slot" in x}
    emu.close()


@pytest.mark.parametrize("block", BLOCKS)
def test_misses_are_listed_and_nothing_is_written(lib, block):
    G = 24
    rng = np.random.default_rng(200 + block)
    ring, cap, head, bounds = edge_ring(rng, G)
    names = {g: b"g%d" % g for g in range(G) if g != 5}
    versions = {g: 0 for g in range(G)}
    emu = Emu(lib, G, names, versions)
    full = make_meta(requests_of(ring, cap, head, 0), rng)
    partial = full[rng.random(len(full)) < 0.9]
    for meta in (partial, full, full[:0]):
        want = expected_misses(ring, cap, head, 0, names, meta)
        assert want
        rc, f, out, miss, sz = emu.frame(ring, cap, head, 0, meta, block)
        assert rc == abi.GPX_ENOENT and f == 0 and sz[:2] == (0, 0) and np.all(out == 0xCD)
        assert [(int(m["gid"]), int(m["kind"]), int(m["req_id"])) for m in miss[: sz[2]]] == want
        # too small a list: the count is reported, nothing written
        rc, f, out, miss, sz2 = emu.frame(ring, cap, head, 0, meta, block, caps=(1 << 20, 1 << 16, len(want) - 1))
        assert rc == abi.GPX_ERANGE and sz2[2] == len(want) and np.all(miss.view(np.uint8) == 0xCD)
    # the name comes, the table is completed: the frames are LogDrainer's
    names[5] = b"g5"
    emu.close()
    emu = Emu(lib, G, names, versions)
    check_same(emu, ring, cap, head, 0, names, versions, full, block)
    emu.close()


def test_sizes_order_and_empty_ranges(lib):
    G = 24
    rng = np.random.default_rng(7)
    ring, cap, head, bounds = edge_ring(rng, G)
    names = {g: b"g%d" % g for g in range(G)}
    versions = {g: 0 for g in range(G)}
    emu = Emu(lib, G, names, versions)
    meta = make_meta(requests_of(ring, cap, head, 0), rng)
    rc, f, out, _, sz = emu.frame(ring, cap, head, 0, meta)
    assert rc == 0 and sz[0] > 10000 and sz[2] == 0
    for caps in ((sz[0] - 1, sz[1], 0), (sz[0], sz[1] - 1, 0)):  # GPX_ERANGE: the sizes, nothing written
        rc, f, out, _, sz2 = emu.frame(ring, cap, head, 0, meta, caps=caps)
        assert rc == abi.GPX_ERANGE and sz2[:2] == sz[:2] and f == 0 and np.all(out == 0xCD)
    for bad in (meta[::-1], np.concatenate([meta[:3], meta[2:]])):  # unsorted, a duplicate
        rc, f, out, _, _ = emu.frame(ring, cap, head, 0, bad, caps=sz)
        assert rc == abi.GPX_EINVAL and f == 0 and np.all(out == 0xCD)
    for b in bounds:  # empty ranges, at every segment boundary
        rc, f, out, _, sz3 = emu.frame(ring, cap, b, b, meta)
        assert rc == 0 and f == b and sz3 == (0, 0, 0)
    rc, f, _, _, _ = emu.frame(ring, cap, head, 16, meta)  # not a segment boundary
    assert rc == abi.GPX_EINVAL and f == 16
    rc, f, _, _, _ = emu.frame(ring, cap, head + 2 * cap, 0, meta)  # overwritten
    assert rc == abi.GPX_ERANGE and f == 0
    emu.close()


def test_journal_frame_kernels_are_clean_under_asan_and_ubsan():
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_journal_frames.py"), "-k", "not asan"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
