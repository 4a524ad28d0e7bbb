"""CPU: gpx_journal_compact_device's kernels (gigapaxos_b200/csrc/gpx_journal_gc.cuh) and its host sequence
(journal_compact in gpx_wire_seq.h) compiled for the host (tests/emu/journal_gc_emu.cpp), against journal.compact_files
on the same files: the statuses, counts and compacted bytes are identical, at block sizes 1, 7 and 64.  The journals
are LogDrainer's frames of the oracle engine's rings (fused rounds, batched slots, partial ACCEPTs, a view change's
PREPAREs, and a small ring that wraps), rolled into several files, and hand-laid files for the edges: GC slots, slots
and ballots across the int32 wrap, the getSlot divergence, unknown names, stale versions and groups that are not live,
STOP decisions, batched ACCEPTs, escaped names, a torn tail, files that stay, files that empty, and malformed frames.
Compaction keeps what recovery reads: replay_accepts / replay_decisions above each group's GC slot and each group's
highest PREPARE.  Also once more under AddressSanitizer + UBSan."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from gigapaxos_b200 import journal, wire
from helpers import ROOT, abi, emu_library, ptr, relay_into_small_ring
from test_journal_frames import hard_names, log_drainer, make_meta, oracle_ring, requests_of
from test_log_find import logged_engine

BLOCKS = [1, 7, 64]
I32 = (-(1 << 31), (1 << 31) - 1)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = emu_library(tmp_path_factory, "journal_gc_emu")
    lib.emu_jgc_new.restype = C.c_void_p
    lib.emu_jgc_new.argtypes = [C.c_uint32]
    lib.emu_jgc_free.argtypes = [C.c_void_p]
    lib.emu_jgc_names.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emu_jgc_compact.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                    C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_uint32]
    lib.emu_jgc_index.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    return lib


def index(lib, buf, base=0, cap=None):
    """gpx_journal_index's walk -> (rc, starts, end)"""
    arr = np.frombuffer(buf, np.uint8) if buf else np.zeros(1, np.uint8)
    cap = len(buf) // 4 + 1 if cap is None else cap
    starts = np.zeros(max(cap, 1), np.uint32)
    n, end = np.zeros(1, np.uint32), np.zeros(1, np.uint64)
    rc = lib.emu_jgc_index(ptr(arr), len(buf), base, ptr(starts), cap, ptr(n), ptr(end))
    return rc, starts[: min(int(n[0]), cap)], int(end[0])


class Gc:
    """one lane's world in the emulator: the name table and the live groups, then calls on files"""

    def __init__(self, lib, G, names, versions, live=None):
        self.lib, self.h, self.G = lib, lib.emu_jgc_new(G), G
        self.names, self.versions = names, versions
        self.live = live if live is not None else {g: True for g in names}
        gids = np.array(sorted(names), np.uint32)
        staged = np.zeros((len(gids), 128), np.uint8)
        for k, g in enumerate(gids):
            staged[k, 0] = len(names[int(g)])
            staged[k, 1: 1 + len(names[int(g)])] = np.frombuffer(names[int(g)], np.uint8)
        ver = np.array([versions[int(g)] for g in gids], np.int32)
        lv = np.array([1 if self.live[int(g)] else 0 for g in gids], np.uint8)
        lib.emu_jgc_names(self.h, len(gids), ptr(gids), ptr(staged), ptr(ver), ptr(lv))
        self.by_name = {(names[g].decode("iso-8859-1"), versions[g]): g for g in names if self.live[g]}

    def close(self):
        self.lib.emu_jgc_free(self.h)

    def gc_slot_of(self, gc):
        def f(pid, ver):
            g = self.by_name.get((pid, ver))
            return None if g is None else int(gc[g])
        return f

    def compact(self, blobs, gc, last_readonly=True, block=64, starts=None, file_off=None, caps=None):
        """-> (rc, [CompactedFile] or None, bad indices, sizes, untouched outputs)"""
        data = np.frombuffer(b"".join(blobs) or b"\0", np.uint8).copy()
        n_bytes = sum(len(b) for b in blobs)
        if file_off is None:
            file_off = np.zeros(len(blobs) + 1, np.uint32)
            file_off[1:] = np.cumsum([len(b) for b in blobs])
        file_off = np.ascontiguousarray(file_off, np.uint32)
        if starts is None:
            starts = np.concatenate([index(self.lib, b, int(o))[1] for b, o in zip(blobs, file_off[:-1])] or
                                    [np.zeros(0, np.uint32)])
        starts = np.ascontiguousarray(starts, np.uint32)
        gc = np.ascontiguousarray(gc, np.int32)
        k = len(file_off) - 1

        def call(sz):
            out = np.full(max(int(sz[0]), 1), 0xCD, np.uint8)
            files = np.zeros(max(k, 1), abi.journal_file_dtype)
            files.view(np.uint8)[:] = 0xCD
            bad = np.full(max(int(sz[1]), 1), 0xCDCDCDCD, np.uint32)
            rc = self.lib.emu_jgc_compact(self.h, ptr(data), n_bytes, ptr(file_off), k, ptr(starts) if len(starts)
                                          else None, len(starts), ptr(gc), len(gc), 1 if last_readonly else 0,
                                          ptr(out), ptr(files), ptr(bad), ptr(sz), block)
            return rc, out, files, bad
        sz = np.array(caps if caps is not None else (0, 0), np.uint64)
        rc, out, files, bad = call(sz)
        if caps is None and rc == abi.GPX_ERANGE:
            rc, out, files, bad = call(sz)
        sizes = tuple(int(x) for x in sz)
        if rc != 0:
            untouched = bool(np.all(out == 0xCD) and np.all(files.view(np.uint8) == 0xCD))
            return rc, None, bad[: sizes[1]].tolist(), sizes, untouched
        assert np.all(out[sizes[0]:] == 0xCD)
        res = [journal.CompactedFile(int(x["status"]),
                                     out[int(x["out_off"]): int(x["out_off"]) + int(x["out_bytes"])].tobytes()
                                     if int(x["status"]) == journal.JGC_COMPACTED else None,
                                     int(x["kept"]), int(x["dropped"]), int(x["unresolved"])) for x in files[:k]]
        assert sum(int(x["out_bytes"]) for x in files[:k]) == sizes[0]
        return rc, res, [], sizes, True


def write_files(tmp_path, blobs, tag="f"):
    paths = []
    for i, b in enumerate(blobs):
        p = tmp_path / f"{tag}{i:03d}"
        p.write_bytes(b)
        paths.append(str(p))
    return paths


def check_same(gc_emu, tmp_path, blobs, gc, block, last_readonly=True, tag="f"):
    paths = write_files(tmp_path, blobs, tag)
    want = journal.compact_files(paths, gc_emu.gc_slot_of(gc), last_readonly)
    rc, got, _, _, _ = gc_emu.compact(blobs, gc, last_readonly, block)
    assert rc == 0, rc
    assert got == want
    return paths, want


def roll(data, rng, n_files):
    """one journal's frames rolled into n_files files at frame boundaries (some of them empty)"""
    offs = [p for p, _ in journal._frames(data)[0]] + [len(data)]
    cuts = sorted(rng.choice(offs, size=n_files - 1, replace=True).tolist())
    bounds = [0] + cuts + [len(data)]
    return [data[a:b] for a, b in zip(bounds[:-1], bounds[1:])]


def gc_slots_for(blobs, gc_emu, rng):
    """per gid a GC slot that drops about half its frames: a slot of its own frames, -1, or one far off"""
    slots = {}
    for b in blobs:
        for _, pkt in journal._frames(b)[0]:
            v = journal.parse_packet(pkt)
            g = gc_emu.by_name.get((v["paxos_id"], v["version"]))
            if g is not None:
                slots.setdefault(g, []).append(v["first_undecided_slot"] if v["kind"] == "PREPARE" else v["slot"])
    gc = np.full(gc_emu.G, -1, np.int32)
    for g, s in slots.items():
        c = rng.random()
        gc[g] = (sorted(s)[len(s) // 2] if c < 0.7 else -1 if c < 0.8 else max(s) if c < 0.9 else I32[0])
    return gc


def replay_above(paths, gc_emu, gc):
    """what recovery reads: per paxosID, ACCEPTs and DECISIONs above the group's GC slot, and the ballots of the
    PREPAREs above it"""
    acc, dec = journal.replay_accepts(paths), journal.replay_decisions(paths)
    f = gc_emu.gc_slot_of(gc)

    def above(d):
        out = {}
        for pid, per in d.items():
            for s, v in per.items():
                g = f(pid, v["version"])
                if g is None or journal._jsub(s, g) > 0:
                    out.setdefault(pid, {})[s] = v
        return out
    prep = {}
    for p in paths:
        for pkt in journal.read_journal(p):
            v = journal.parse_packet(pkt)
            g = f(v["paxos_id"], v["version"]) if v["kind"] == "PREPARE" else None
            if v["kind"] == "PREPARE" and (g is None or journal._jsub(v["first_undecided_slot"], g) > 0):
                prep.setdefault(v["paxos_id"], set()).add((v["bnum"], v["bcoord"]))
    return above(acc), above(dec), prep


def apply(paths, results):
    for p, r in zip(paths, results):
        if r.status == journal.JGC_COMPACTED:
            with open(p, "wb") as f:
                f.write(r.data)
        elif r.status == journal.JGC_EMPTY:
            os.remove(p)
    return [p for p, r in zip(paths, results) if r.status != journal.JGC_EMPTY]


# ---- the oracle engine's journals ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("block", BLOCKS)
def test_oracle_journals_compact_as_compact_files_does(oracle_lib, lib, block, tmp_path):
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed=block)
    rng = np.random.default_rng(block)
    names = hard_names(G, rng)
    versions = {g: int(rng.choice([0, 1, I32[0], I32[1]])) for g in range(G)}
    gce = Gc(lib, G, names, versions)
    dropped = kept = 0
    for lane in range(3):
        ring, cap, head = oracle_ring(eng, lane)
        meta = make_meta(requests_of(ring, cap, head, 0), rng)
        data, _ = log_drainer(ring, cap, head, 0, names, versions, meta)
        kinds = {journal.parse_packet(p)["kind"] for _, p in journal._frames(data)[0]}
        assert kinds == {"ACCEPT", "DECISION", "PREPARE"}
        blobs = roll(data, rng, 6)
        gc = gc_slots_for(blobs, gce, rng)
        before = replay_above(write_files(tmp_path, blobs, f"b{lane}_"), gce, gc)
        paths, res = check_same(gce, tmp_path, blobs, gc, block, tag=f"l{lane}_")
        dropped += sum(r.dropped for r in res)
        kept += sum(r.kept for r in res)
        # recovery reads the same records above each GC slot, and every group keeps its highest PREPARE
        after_paths = apply(paths[:-1], res[:-1]) + paths[-1:]
        acc, dec, prep = replay_above(after_paths, gce, gc)
        assert (acc, dec) == before[:2]
        for pid, ballots in before[2].items():
            assert max(ballots) in prep.get(pid, set())
        # without a read-only last file every file is compacted
        check_same(gce, tmp_path, blobs, gc, block, last_readonly=False, tag=f"w{lane}_")
    assert dropped > 200 and kept > 200
    gce.close()
    eng.close()


@pytest.mark.parametrize("block", BLOCKS)
def test_a_journal_from_a_ring_that_wraps(oracle_lib, lib, block, tmp_path):
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed=20 + block, rounds=9)
    rng = np.random.default_rng(block)
    names = {g: b"NoopPaxosApp%d" % g for g in range(G)}
    versions = {g: 0 for g in range(G)}
    gce = Gc(lib, G, names, versions)
    for lane in range(3):
        buf, hs = eng.log_read(lane), heads[lane]
        cap = 1 << int(np.ceil(np.log2(2.2 * max(b - a for a, b in zip(hs[:-1], hs[1:])))))
        ring, head, _, call_pos = relay_into_small_ring(buf, hs, cap)
        assert head > 2 * cap
        first = next(i for i, p in enumerate(call_pos) if head - p <= cap)
        meta = make_meta(requests_of(ring, cap, head, call_pos[first]), rng)
        data, _ = log_drainer(ring, cap, head, call_pos[first], names, versions, meta)
        blobs = roll(data, rng, 4)
        check_same(gce, tmp_path, blobs, gc_slots_for(blobs, gce, rng), block, tag=f"l{lane}_")
    gce.close()
    eng.close()


# ---- hand-laid files ------------------------------------------------------------------------------------------------------
def frame(pkt):
    return struct.pack(">i", len(pkt)) + pkt


def accept(pid, ver, slot, bnum, bcoord, req_id=7, value=b"v", batched=(), stop=False):
    subs = tuple(wire.Request(pid, ver, r, b"s%d" % r, stop=st, entry_replica=101, entry_time=5) for r, st in batched)
    req = wire.Request(pid, ver, req_id, value, stop=stop, entry_replica=100, entry_time=1760000000000, batched=subs)
    return frame(wire.encode_accept(req, slot, bnum, bcoord, False, slot - 1, 100))


def decision(pid, ver, slot, bnum, bcoord, stop=False):
    return frame(journal.decision_json(pid, ver, slot, bnum, bcoord, -1, 9, 100, 1 << 40, stop=stop))


def prepare(pid, ver, bnum, bcoord, first):
    return frame(journal.prepare_json(pid, ver, bnum, bcoord, first))


def packets(data):
    return [p for _, p in journal._frames(data)[0]]


def hand_world(lib):
    names = {0: b"g0", 1: b"g1", 2: b'we"ird\\\x01\xe9\x7f/', 3: b"wrap", 4: b"paused", 5: b"prep"}
    versions = {0: 0, 1: 3, 2: I32[0], 3: 0, 4: 0, 5: 0}
    live = {g: g != 4 for g in names}
    gce = Gc(lib, 8, names, versions, live)
    gc = np.array([10, 10, 5, I32[1] - 2, 0, 10, -1, -1], np.int32)
    return gce, gc


@pytest.mark.parametrize("block", BLOCKS)
def test_hand_laid_edges(lib, block, tmp_path):
    gce, gc = hand_world(lib)
    weird = b'we"ird\\\x01\xe9\x7f/'.decode("iso-8859-1")
    f0 = b"".join([
        accept("g0", 0, 10, 1, 100),        # at the GC slot: dropped
        accept("g0", 0, 11, 3, 100),        # getSlot divergence: ballot number 3 <= gcSlot 10 < slot 11: kept
        decision("g0", 0, 9, 2, 100, stop=True),  # below: dropped
        decision("g0", 0, 12, 2, 101, stop=True),  # STOP above: kept
        accept("g1", 3, 11, 1, 100, batched=[(8, False), (9, True)]),  # batched, above: kept
        accept("g1", 2, 1, 1, 100),         # stale version: kept
        accept("nobody", 0, 1, 1, 100),     # unknown name: kept
        accept("paused", 0, -5, 1, 100),    # not live: kept
        decision(weird, I32[0], 5, 1, 100),  # escaped name at its GC slot: dropped
        decision(weird, I32[0], 6, 1, 100),  # kept
        accept("wrap", 0, I32[1] - 2, 1, 100),  # at the GC slot: dropped
        accept("wrap", 0, I32[1], 1, 100),  # above: kept
        accept("wrap", 0, I32[0], 1, 100),  # wrapped above: kept
        accept("wrap", 0, I32[0] + 5, 1, 100),
        decision("wrap", 0, I32[1] - 100, 1, 100),  # below: dropped
    ])
    f1 = b"".join([  # every frame dropped: the file empties
        accept("g0", 0, 3, 1, 100), decision("g0", 0, 10, 1, 100), decision(weird, I32[0], -3, 1, 100)])
    f2 = b"".join([  # all needed: unchanged
        accept("g0", 0, 20, 5, 100), decision("g1", 3, 30, 5, 100), prepare("nobody", 0, 1, 1, 0)])
    f3 = b"".join([  # PREPAREs against the indexed ballots of their group, across the wrap
        prepare("prep", 0, I32[1] - 1, 100, 20),  # an indexed ACCEPT at bnum INT32_MIN + 1 is higher: dropped
        accept("prep", 0, 21, I32[0] + 1, 100),
        prepare("prep", 0, I32[0] + 1, 99, 20),  # equal bnum, coordinator 100 - 99 > 0: dropped
        prepare("prep", 0, I32[0] + 1, 100, 20),  # equal ballot: the highest, kept
        prepare("prep", 0, I32[0] + 2, 100, 5),  # at the GC slot: dropped
        prepare("g0", 0, 9, 100, 11),  # g0's entries above have bnums 3, 2, 5: 9 is the highest, kept
        prepare("g0", 0, 2, 100, 11),  # dropped
    ])
    f4 = accept("g0", 0, 4, 1, 100) + accept("g0", 0, 40, 1, 100) + b"\x00\x00\x01\x00torn"  # torn tail
    f5 = decision("prep", 0, 25, I32[0] + 1, 100) + accept("g0", 0, 1, 1, 100)  # read-only last
    blobs = [f0, f1, f2, f3, f4, f5]
    paths, res = check_same(gce, tmp_path, blobs, gc, block)
    st = [r.status for r in res]
    assert st == [journal.JGC_COMPACTED, journal.JGC_EMPTY, journal.JGC_UNCHANGED, journal.JGC_COMPACTED,
                  journal.JGC_TORN, journal.JGC_UNCHANGED]
    assert [(r.kept, r.dropped) for r in res] == [(10, 5), (0, 3), (3, 0), (3, 4), (2, 0), (2, 0)]
    assert [r.unresolved for r in res] == [3, 0, 1, 0, 0, 0]
    kept0 = [journal.parse_packet(p) for p in packets(res[0].data)]
    assert (kept0[0]["slot"], kept0[0]["bnum"]) == (11, 3)  # the divergence case is kept
    kept3 = [journal.parse_packet(p) for p in packets(res[3].data)]
    assert [(v["kind"], v["bnum"], v["bcoord"]) for v in kept3] == [
        ("ACCEPT", I32[0] + 1, 100), ("PREPARE", I32[0] + 1, 100), ("PREPARE", 9, 100)]
    # the read-only flag off: the last file is compacted too
    _, res2 = check_same(gce, tmp_path, blobs, gc, block, last_readonly=False, tag="w")
    assert res2[-1].status == journal.JGC_COMPACTED and res2[-1].kept == 1
    # no files, one empty file, files without frames
    rc, got, _, sizes, _ = gce.compact([b""], gc, True, block)
    assert rc == 0 and got == [journal.CompactedFile(journal.JGC_UNCHANGED, None, 0, 0, 0)]
    rc, got, _, _, _ = gce.compact([b"", b"\x00\x00", b""], gc, True, block)
    assert rc == 0 and [r.status for r in got] == [journal.JGC_EMPTY, journal.JGC_TORN, journal.JGC_UNCHANGED]
    gce.close()


def test_errors_write_nothing_but_the_list(lib, tmp_path):
    gce, gc = hand_world(lib)
    good = accept("g0", 0, 11, 1, 100)
    bad_json = [frame(b'{"type":90,"PT":6,"ID":"g0","V":0,"B":"1:100","S":x}'),
                frame(b'{"type":91,"PT":6,"ID":"g0","V":0,"B":"1:100","GC_S":-1,"S":3,"QID":1,"ET":1,"E":1}'),
                frame(b'{"type":90,"PT":7,"ID":"g0","V":0,"B":"1:100","PREP_MIN":3}'),
                frame(b'{"type":90,"PT":2,"ID":"g0","V":0,"B":"1-100","PREP_MIN":3}'),
                frame(b'{"type":90,"PT":2,"ID":"g0","V":0,"B":"1:100"}'),
                frame(b'{"type":90,"PT":2,"ID":"g0","V":0,"B":"1:100","PREP_MIN":3} x'),
                frame(b'{"type":90,"PT":6,"ID":"g0","V":0,"B":"1:100","S":3}'),
                frame(good[4:-1]), frame(good[4:] + b"\x00"), frame(b""),
                frame(wire.encode_batched_accept_reply("g0", 0, 100, 1, 100, 1, 0, 1, [1], [1]))]
    for k, b in enumerate(bad_json):
        blobs = [good + b + good, good]
        with pytest.raises(ValueError):
            journal.compact_files(write_files(tmp_path, blobs, "e%d_" % k), gce.gc_slot_of(gc))
        rc, got, bad, sizes, untouched = gce.compact(blobs, gc)
        assert (rc, bad, sizes[0], untouched) == (abi.GPX_EINVAL, [1], 0, True), k
    data = [good + good, good]
    # a length that disagrees with the next start, a start that skips the file's first frame, one past the input
    for starts in ([0, len(good) - 1, 2 * len(good)], [len(good), 2 * len(good)], [0, len(good), 2 * len(good) + 1]):
        rc, _, bad, _, untouched = gce.compact(data, gc, starts=starts)
        assert rc == abi.GPX_EINVAL and untouched and bad, starts
    rc, _, bad, _, _ = gce.compact(data, gc, starts=[0, len(good) - 1, 2 * len(good)])
    assert bad == [0, 1]
    rc, _, bad, _, untouched = gce.compact(data, gc, file_off=[0, 2 * len(good) + 4, 3 * len(good)])
    assert rc == abi.GPX_EINVAL and untouched  # a frame overruns its file
    rc, _, bad, _, untouched = gce.compact(data, gc, file_off=[0, 3 * len(good), 2 * len(good)])
    assert rc == abi.GPX_EINVAL and untouched and bad == []  # file_off not ascending
    # capacities: GPX_ERANGE reports the sizes and writes nothing
    blobs = [good + accept("g0", 0, 3, 1, 100), good]
    rc, _, _, sizes, untouched = gce.compact(blobs, gc, caps=(len(good) - 1, 0))
    assert (rc, sizes, untouched) == (abi.GPX_ERANGE, (len(good), 0), True)
    rc, _, bad, sizes, untouched = gce.compact([good + frame(b"{")], gc, caps=(0, 0))
    assert (rc, sizes, untouched) == (abi.GPX_ERANGE, (0, 1), True)
    rc, _, _, _, _ = gce.compact(blobs, gc[:5])
    assert rc == abi.GPX_EINVAL  # a GC slot per group is needed
    gce.close()


def test_index_walks_as_read_journal_does(lib, tmp_path):
    frames = [accept("g0", 0, s, 1, 100) for s in range(5)] + [decision("g0", 0, 9, 1, 100)]
    data = b"".join(frames)
    rc, starts, end = index(lib, data, 100)
    offs = np.cumsum([0] + [len(f) for f in frames[:-1]]) + 100
    assert rc == 0 and starts.tolist() == offs.tolist() and end == len(data)
    for tail in (b"\x00\x00\x00", b"\x00\x00\x00\x09abc", b"\xff\xff\xff\xff", b"\x80\x00\x00\x00xyz"):
        rc, s2, end = index(lib, data + tail)
        p = tmp_path / "t"
        p.write_bytes(data + tail)
        assert rc == 0 and len(s2) == len(list(journal.read_journal(str(p)))) == len(frames) and end == len(data)
    rc, s3, _ = index(lib, data, 0, cap=3)
    assert rc == abi.GPX_ERANGE and s3.tolist() == (offs[:3] - 100).tolist()
    rc, _, _ = index(lib, data, (1 << 32) - 10)
    assert rc == abi.GPX_EINVAL


def test_emulated_journal_gc_is_clean_under_asan_and_ubsan():
    if os.environ.get("GPX_EMU_SANITIZE"):
        pytest.skip("already the sanitized child")
    asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not asan or not os.path.exists(asan) or not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("no libasan / CUDA headers")
    env = dict(os.environ, GPX_EMU_SANITIZE="1", LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")
    r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "hand_laid or errors or index or (oracle and 7)"],
                       capture_output=True, text=True, env=env, cwd=ROOT, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert " passed" in r.stdout and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
