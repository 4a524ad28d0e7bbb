"""gpx_log_find: the journal's index as a scan of the log ring (AbstractPaxosLogger.getLoggedDecisions :582 /
getLoggedAccepts :568 in the journaling form, SQLPaxosLogger.getLoggedFromMessageLog :3674-3756: per wanted slot the
entry logged LAST).

CPU: the oracle's entry point against a walk of the same ring bytes in Python (abi.parse_log), and the CUDA kernels' own
source (gigapaxos_b200/csrc/gpx_logfind.cuh) compiled for the host (tests/emu) on the oracle engine's real ring bytes --
as they lie, and re-laid into a small ring that wraps (stale laps, skipped tails) the way the device lays them.  The GPU
test is in tests/test_zz_phase1b_gpu.py."""
import ctypes as C

import numpy as np
import pytest

# GPX_EMU_SANITIZE=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) python -m pytest ... : the emulated kernels under
# AddressSanitizer + UBSan (every heap buffer numpy hands them gets red zones; so do their local arrays)
from helpers import Engine, abi, emu_library, group_descs, make_config, make_requests, ptr, relay_into_small_ring

NODES = [100, 101, 102]


def logged_engine(lib, G=40, seed=1, rounds=5, **cfg):
    """an engine with a varied journal: fused rounds, phase-by-phase rounds with partial delivery, batched slots, a view
    change (PREPARE segments, the same slot accepted again under a higher ballot).  Returns (engine, per-lane list of the
    ring head after every call)."""
    kw = dict(max_groups=G, max_batch_recs=4096, max_batch_payload=1 << 20)
    kw.update(cfg)
    eng = Engine(lib, make_config(lib, **kw))
    eng.create_groups(group_descs(G))
    heads = [[0] for _ in range(3)]

    def mark():
        for l in range(3):
            h = eng.log_head(l)
            if h != heads[l][-1]:
                heads[l].append(h)

    rng = np.random.default_rng(seed)
    gids = np.arange(G, dtype=np.uint32)
    for r in range(rounds):
        sel = gids[rng.random(G) < 0.8]
        per = np.where(rng.random(len(sel)) < 0.2, 2, 1)
        reqs, pay = make_requests(np.repeat(sel, per), payload_len=3 + r, seed=seed, round_no=r)
        eng.round(reqs, pay)
        mark()
    rows0 = eng.dump_rows(gids, 0)
    coord = np.array([NODES.index(int(x)) for x in rows0["acc_bcoord"]])
    for k, reach in enumerate((0b011, 0b110)):  # ACCEPTs that reach only some acceptors and are never decided
        reqs, pay = make_requests(gids, payload_len=9 + k, seed=seed + 1, round_no=k)
        reqs["flags"] = coord << 8
        reqs["entry_node"] = np.array(NODES)[coord]
        acc, blob, st = eng.propose(reqs, pay)
        acc["dst_mask"] = reach
        eng.handle_accepts(acc, blob)
        mark()
    # the next node takes over every group: PREPAREs are logged, then the carried-over slots are accepted AGAIN under the
    # new ballot (the later entry must win) and decided
    from gigapaxos_b200.paxos_manager import NoopPaxosApp, PaxosManager, _Instance
    pm = PaxosManager(eng, [NoopPaxosApp() for _ in NODES], NODES, device_phase1b=lib.has("handle_prepare_replies"))
    for i in range(G):  # adopt the groups created above (group_descs names them NoopPaxosApp<i>, gid i)
        pm.instances[f"NoopPaxosApp{i}"] = _Instance(i, 0, NODES)
        pm.gid_name[i] = f"NoopPaxosApp{i}"
    pm.next_gid = G
    for c in range(3):
        names = [f"NoopPaxosApp{i}" for i in range(G) if coord[i] == c]
        won = pm.runForCoordinators(names, (c + 1) % 3)
        assert all(won.values())
        mark()
    return eng, heads


def test_body_pos_maps_a_ring_offset_to_the_live_position(oracle_lib):
    """the kernels keep a pvalue's frame_ref as its body's offset inside the ring / 16; PaxosManager._body_pos turns it
    back into the one live absolute position -- every 16-byte boundary of [head - ring, head), both ends included, on a
    log that has wrapped twice"""
    from gigapaxos_b200.paxos_manager import NoopPaxosApp, PaxosManager
    G, cap = 40, 1 << 16
    eng = Engine(oracle_lib, make_config(oracle_lib, max_groups=G, max_batch_recs=4096, max_batch_payload=1 << 20,
                                         log_ring_bytes=cap))
    eng.create_groups(group_descs(G))
    r = 0
    while eng.log_head(0) < 2 * cap:
        reqs, pay = make_requests(np.arange(G, dtype=np.uint32), payload_len=40, seed=3, round_no=r)
        eng.round(reqs, pay)
        r += 1
    head = eng.log_head(0)
    assert head % 16 == 0
    pm = PaxosManager(eng, [NoopPaxosApp() for _ in NODES], NODES)
    assert pm._body_pos(0, ((head - cap) % cap) // 16) == head - cap  # exactly one lap behind: still live
    assert pm._body_pos(0, ((head - 16) % cap) // 16) == head - 16
    for p in range(head - cap, head, 16):
        assert pm._body_pos(0, (p % cap) // 16, head) == p
    eng.close()


def python_find(eng, lane, wants, start=0):
    """the expected answer from a walk of the ring bytes in log order"""
    buf = eng.log_read(lane, start)
    out = np.zeros((len(wants), abi.GPX_LOG_SPAN), dtype=abi.log_hit_dtype)
    out["decision"]["flags"] = abi.F_VOID
    out["accept"]["flags"] = abi.F_VOID
    idx = {int(w["gid"]): i for i, w in enumerate(wants)}
    for hdr, imgs, payload, pay_off in abi.parse_log(buf):
        rec, typ = int(hdr["rec_bytes"]), int(hdr["type"])
        if not (rec == 48 or (rec == 32 and typ == abi.F_DECISION)):
            continue
        for im in imgs:
            if int(im["flags"]) & abi.F_VOID or int(im["gid"]) not in idx:
                continue
            i = idx[int(im["gid"])]
            k = (int(im["slot"]) - int(wants[i]["min_slot"]) + (1 << 31)) % (1 << 32) - (1 << 31)
            if k < 0 or k >= int(wants[i]["n_slots"]):
                continue
            if rec == 48:
                out[i, k]["accept"] = im
                out[i, k]["blob_pos"] = start + pay_off + int(im["payload_off"])
            else:
                for f in abi.decision_dtype.names:
                    out[i, k]["decision"][f] = im[f]
    return out


def random_wants(G, rng, max_slot=12):
    gids = np.sort(rng.choice(G + 3, size=int(rng.integers(1, G)), replace=False)).astype(np.uint32)  # some never logged
    w = np.zeros(len(gids), dtype=abi.log_want_dtype)
    w["gid"], w["min_slot"] = gids, rng.integers(0, max_slot, size=len(gids))
    w["n_slots"] = rng.integers(0, abi.GPX_LOG_SPAN + 1, size=len(gids))
    return w


@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_log_find_equals_a_walk_of_the_ring(oracle_lib, seed):
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed)
    rng = np.random.default_rng(seed)
    found = 0
    for lane in range(3):
        for start in (0, heads[lane][len(heads[lane]) // 2]):
            wants = random_wants(G, rng)
            got, want = eng.log_find(lane, wants, start), python_find(eng, lane, wants, start)
            assert got.tobytes() == want.tobytes()
            hit_d = (got["decision"]["flags"] & abi.F_VOID) == 0
            hit_a = (got["accept"]["flags"] & abi.F_VOID) == 0
            found += int(hit_d.sum()) + int(hit_a.sum())
            for i, k in np.argwhere(hit_a)[:3]:  # the blob position leads to the request body the ACCEPT was logged with
                a = got[i, k]["accept"]
                body = bytes(eng.log_read(lane, int(got[i, k]["blob_pos"]), int(a["payload_len"])))
                assert len(body) == int(a["payload_len"]) > 0
    assert found > 100
    with pytest.raises(abi.GpxError):
        bad = np.zeros(2, dtype=abi.log_want_dtype)
        bad["gid"] = [3, 3]
        eng.log_find(0, bad)
    # the same slot accepted under two ballots: the entry logged last (the higher ballot's) is the one found
    w = np.zeros(G, dtype=abi.log_want_dtype)
    w["gid"], w["min_slot"], w["n_slots"] = np.arange(G), 0, 16
    h = eng.log_find(0, w)
    row0 = eng.dump_rows(np.arange(G, dtype=np.uint32), 0)
    ok = (h["accept"]["flags"] & abi.F_VOID) == 0
    assert np.any(h["accept"]["bnum"][ok] == row0["acc_bnum"].max())


# ---- the CUDA kernels' own source on the host, driven by the engine's own sequences (gpx_state_seq.h) ----------------------
@pytest.fixture(scope="module")
def emu_lib(tmp_path_factory):
    lib = emu_library(tmp_path_factory, "logfind_emu")
    lib.emu_log_find.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                 C.c_void_p, C.c_uint32, C.c_uint32]
    lib.emu_log_gather.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                   C.c_uint64, C.c_uint32]
    return lib


def emu_find(emu_lib, ring, cap, head, start, lane, wants, grid=3, block=64, rc=1, error=None):
    """gpx_log_find on the ring image; rc: 1 (k_log_dir's launch) or the GPX_* error expected, with `error` in its
    message"""
    hits = np.zeros((len(wants), abi.GPX_LOG_SPAN), dtype=abi.log_hit_dtype)
    hits.view(np.uint8)[:] = 0xCD
    assert emu_lib.emu_log_find(ptr(ring), cap, head, start, lane, len(wants), ptr(wants), ptr(hits), grid, block) == rc
    if error:
        assert error in emu_lib.emu_last_error().decode()
    return hits


@pytest.mark.parametrize("seed,grid,block", [(3, 3, 64), (4, 1, 1), (5, 7, 256)])
def test_kernel_source_on_the_host_equals_oracle(oracle_lib, emu_lib, seed, grid, block):
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed)
    rng = np.random.default_rng(seed)
    for lane in range(3):
        head = eng.log_head(lane)
        cap = 1 << int(np.ceil(np.log2(head + 64)))
        ring = np.zeros(cap, dtype=np.uint8)
        ring[:head] = eng.log_read(lane)
        for start in (0, heads[lane][len(heads[lane]) // 3]):
            wants = random_wants(G, rng)
            want = eng.log_find(lane, wants, start)
            got = emu_find(emu_lib, ring, cap, head, start, lane, wants, grid=grid, block=block)
            assert got.tobytes() == want.tobytes()
    # bytes that were overwritten: reported, nothing found
    wants = random_wants(G, rng)
    got = emu_find(emu_lib, ring, cap, head + 2 * cap, 0, 2, wants, rc=abi.GPX_ERANGE, error="already overwritten")
    assert np.all(got["decision"]["flags"] == abi.F_VOID) and np.all(got["accept"]["flags"] == abi.F_VOID)


def test_more_segments_than_the_directory_holds(emu_lib):
    """the directory holds ring_cap / GPX_SEG_DEC_BYTES(1) + 2 segments, more than any launch of the engine fills the
    ring with; a ring of 64-byte segments that carry no slot (no launch writes those) overfills it: reported, nothing
    found"""
    cap = 1 << 10
    ring = np.zeros(cap, dtype=np.uint8)
    hdr = ring.view(abi.seg_hdr_dtype)
    hdr["magic"], hdr["type"], hdr["rec_bytes"], hdr["ring_off"] = abi.SEG_MAGIC, abi.F_DECISION, 32, np.arange(0, cap, 64)
    wants = np.zeros(1, dtype=abi.log_want_dtype)
    wants["n_slots"] = 4
    got = emu_find(emu_lib, ring, cap, 12 * 64, 0, 0, wants)  # 12 segments: as many as it holds
    assert np.all(got["decision"]["flags"] == abi.F_VOID)
    got = emu_find(emu_lib, ring, cap, 13 * 64, 0, 0, wants, rc=abi.GPX_ERANGE, error="more log segments")
    assert np.all(got["decision"]["flags"] == abi.F_VOID) and np.all(got["accept"]["flags"] == abi.F_VOID)


@pytest.mark.parametrize("seed", [6, 7])
def test_kernel_source_on_a_ring_that_wraps(oracle_lib, emu_lib, seed):
    """stale bytes of earlier laps and the tails skipped at the ring end are not mistaken for segments; what is found is
    what the oracle finds in the calls that are still in the ring"""
    G = 40
    eng, heads = logged_engine(oracle_lib, G, seed, rounds=9)
    rng = np.random.default_rng(seed)
    for lane in range(3):
        buf = eng.log_read(lane)
        hs = heads[lane]
        biggest = max(b - a for a, b in zip(hs[:-1], hs[1:]))
        cap = 1 << int(np.ceil(np.log2(2.2 * biggest)))
        assert cap < hs[-1] / 2  # it really wraps, more than once
        ring, head, seg_map, call_pos = relay_into_small_ring(buf, hs, cap)
        first = next(i for i, p in enumerate(call_pos) if head - p <= cap)  # the oldest call still intact
        assert 0 < first < len(call_pos) - 1
        wants = random_wants(G, rng, max_slot=16)
        want = eng.log_find(lane, wants, hs[first])
        got = emu_find(emu_lib, ring, cap, head, call_pos[first], lane, wants)
        for f in ("decision", "accept"):
            assert got[f].tobytes() == want[f].tobytes(), f
        assert ((want["accept"]["flags"] & abi.F_VOID) == 0).any()
        # blob positions: the same offset inside the same segment, at the segment's new position
        old_segs = np.array(sorted(seg_map))
        for i, k in np.argwhere((want["accept"]["flags"] & abi.F_VOID) == 0):
            ob = int(want[i, k]["blob_pos"])
            seg = int(old_segs[np.searchsorted(old_segs, ob, side="right") - 1])
            assert int(got[i, k]["blob_pos"]) == seg_map[seg] + (ob - seg)
            n = int(want[i, k]["accept"]["payload_len"])
            gp = int(got[i, k]["blob_pos"]) % cap
            assert bytes(ring[gp: gp + n]) == bytes(buf[ob: ob + n])
        # one call too far back: its bytes are gone
        emu_find(emu_lib, ring, cap, head, call_pos[0], lane, wants, rc=abi.GPX_ERANGE, error="already overwritten")


def test_a_header_with_absurd_sizes_is_not_followed(emu_lib):
    """k_log_dir stops at a header whose sizes would move the walk backwards or beyond a lap (no launch writes such a
    segment): reported as corrupt instead of walking on"""
    cap = 1 << 12
    ring = np.zeros(cap, dtype=np.uint8)
    hdr = ring[:64].view(abi.seg_hdr_dtype)[0]
    hdr["magic"], hdr["type"], hdr["n_slots"], hdr["n_valid"], hdr["rec_bytes"], hdr["ring_off"] = abi.SEG_MAGIC, abi.F_DECISION, 1, 1, 32, 0
    wants = np.zeros(1, dtype=abi.log_want_dtype)
    wants["n_slots"] = 4
    for pb in ((1 << 64) - 64, 1 << 40):
        ring[:64].view(abi.seg_hdr_dtype)[0]["payload_bytes"] = pb
        got = emu_find(emu_lib, ring, cap, 2048, 0, 0, wants, rc=abi.GPX_EINVAL, error="`from` is not a segment boundary")
        assert np.all(got["decision"]["flags"] == abi.F_VOID)


# ---- gpx_log_gather: the bodies of a batch of hits in one copy ---------------------------------------------------------------
def test_log_gather_oracle_and_kernel_source(oracle_lib, emu_lib):
    G = 40
    eng, heads = logged_engine(oracle_lib, G, 9)
    w = np.zeros(G, dtype=abi.log_want_dtype)
    w["gid"], w["min_slot"], w["n_slots"] = np.arange(G), 1, 16
    for lane in range(3):
        h = eng.log_find(lane, w).reshape(-1)
        h = h[(h["accept"]["flags"] & abi.F_VOID) == 0]
        assert len(h) > 100
        pos, ln = h["blob_pos"].astype(np.uint64), h["accept"]["payload_len"]
        ln = ln.copy()
        ln[::7] = 0  # some empty ranges in between
        got = eng.log_gather(lane, pos, ln)
        want = [bytes(eng.log_read(lane, int(p), int(n))) if n else b"" for p, n in zip(pos, ln)]
        assert got == want and sum(len(b) for b in got) > 1000
        # the kernel's source on the ring image (re-laid into a ring that wraps: positions modulo the ring size)
        buf = eng.log_read(lane)
        head = len(buf)
        cap = 1 << int(np.ceil(np.log2(head + 64)))
        ring = np.zeros(cap, dtype=np.uint8)
        ring[:head] = buf
        r = np.zeros(len(pos), dtype=abi.log_range_dtype)
        r["pos"], r["len"] = pos, ln
        padded = (ln.astype(np.uint64) + 15) // 16 * 16
        gaps = np.arange(len(r), dtype=np.uint64) % 3 * 16  # bytes between the ranges read as zero
        r["dst_off"] = np.concatenate([[0], np.cumsum(padded + gaps)[:-1]]) + gaps
        top = int(r["dst_off"][-1] + padded[-1])
        out = np.full(top + 64, 0xEE, dtype=np.uint8)
        for block in (1, 64, 256):
            out[:] = 0xEE
            assert emu_lib.emu_log_gather(ptr(ring), cap, head, lane, len(r), ptr(r), ptr(out), len(out), block) == 0
            written = np.zeros(len(out), dtype=bool)
            for o, n, b in zip(r["dst_off"], ln, want):
                assert bytes(out[int(o): int(o) + int(n)]) == b
                written[int(o): int(o) + int(n)] = True
            assert not out[:top][~written[:top]].any()  # gaps and padding are zero
            assert np.all(out[top:] == 0xEE)  # nothing written past the last chunk
    # the range checks, on a ring of 256 bytes whose head has wrapped to 304: each refused, nothing written
    ring = np.arange(256, dtype=np.uint8)
    out = np.full(64, 0xEE, dtype=np.uint8)
    for pos, ln, dst_off, rc, error in ((56, 4, 0, abi.GPX_EINVAL, "16-byte boundary"),
                                        (48, 4, 8, abi.GPX_EINVAL, "16-byte boundary"),
                                        (288, 32, 0, abi.GPX_ERANGE, "outside the live ring bytes"),
                                        (32, 16, 0, abi.GPX_ERANGE, "outside the live ring bytes"),
                                        (240, 32, 0, abi.GPX_ERANGE, "straddles the ring end"),
                                        (256, 16, 64, abi.GPX_ERANGE, "range beyond dst")):
        r = np.zeros(2, dtype=abi.log_range_dtype)
        r["pos"], r["len"], r["dst_off"] = [256, pos], [16, ln], [16, dst_off]
        assert emu_lib.emu_log_gather(ptr(ring), 256, 304, 0, 2, ptr(r), ptr(out), len(out), 7) == rc, error
        assert error in emu_lib.emu_last_error().decode() and np.all(out == 0xEE)
    r["pos"], r["len"], r["dst_off"] = [256, 288], [16, 16], [16, 48]  # both live: [16, 32) and [48, 64), zeros around
    assert emu_lib.emu_log_gather(ptr(ring), 256, 304, 0, 2, ptr(r), ptr(out), len(out), 7) == 0
    assert not out[:16].any() and list(out[16:32]) == list(range(16)) and not out[32:48].any()
    assert list(out[48:]) == list(range(32, 48))
    with pytest.raises(abi.GpxError):
        eng.log_gather(0, [8], [4])  # not on a 16-byte boundary
    with pytest.raises(abi.GpxError):
        eng.log_gather(0, [eng.log_head(0)], [64])  # beyond the head
    assert eng.log_gather(0, [], []) == []
