"""Journal persistence (SURVEY.md 8f rank 1): the log ring drained into Journaler-compatible files
({int32 BE len}{packet}*, SQLPaxosLogger.java:1000-1003: ACCEPTs byteified, DECISIONs as the JSON string of the meta
decision, :1084-1098) and read back the way SQLPaxosLogger's reader walks a file (:685-848)."""
import os
import types

import numpy as np
import pytest

from gigapaxos_b200 import journal, wire
from gigapaxos_b200.paxos_manager import NoopPaxosApp, PaxosManager
from helpers import Engine, abi, group_descs, make_config, make_requests, relay_into_small_ring

NODES = [100, 101, 102]


def run(lib, tmp_path, n_groups=6, rounds=6, **cfg):
    eng = Engine(lib, make_config(lib, max_groups=32, max_batch_recs=1024, max_batch_payload=1 << 18, **cfg))
    pm = PaxosManager(eng, [NoopPaxosApp() for _ in NODES], NODES)
    names = [f"NoopPaxosApp{i}" for i in range(n_groups)]
    pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
    meta = {}
    sent = {}

    def lookup(gid, rid):
        return meta[rid]

    drainers = [journal.LogDrainer(eng, l, journal.Journaler(str(tmp_path) + "/", NODES[l], max_log_file_size=2000),
                                   lookup) for l in range(3)]
    rng = np.random.default_rng(4)
    for r in range(rounds):
        for n in names:
            for _ in range(int(rng.integers(1, 4))):
                val = bytes(rng.integers(97, 123, size=int(rng.integers(1, 30))).astype(np.uint8))
                rid = pm.propose(n, val, entry_node=NODES[r % 3])
                req = pm.outstanding[rid]
                meta[rid] = (n, 0, req.entry_replica, int(req.entry_time * 1000))
                sent[rid] = (n, val)
        pm.run_round()
        for d in drainers:
            d.drain()
    for d in drainers:
        d.j.close()
    return pm, drainers, sent


def check(pm, drainers, sent):
    for l, d in enumerate(drainers):
        assert len(d.j.files) > 1  # rolled at MAX_LOG_FILE_SIZE (rollLogFile :789-812)
        assert all(os.path.basename(f).startswith(f"log.{NODES[l]}.") for f in d.j.files)
        assert os.path.basename(os.path.dirname(d.j.files[0])) == f"paxos_journal.{NODES[l]}"
        seen = {}
        slots = {}
        dslots = {}
        for f in d.j.files:
            assert not os.path.exists(f + ".decisions")  # one journal, no side file
            for pkt in journal.read_journal(f):
                v = journal.parse_packet(pkt)
                if v["kind"] == "ACCEPT":
                    assert pkt[3] == 90 and pkt[7] == 3  # PAXOS_PACKET / ACCEPT (SQLPaxosLogger.toBytes :1090)
                    slots.setdefault(v["paxos_id"], []).append(v["slot"])
                    seen[v["request_id"]] = (v["paxos_id"], v["value"])
                else:
                    assert v["kind"] == "DECISION" and pkt[:1] == b"{"  # the JSON string of the meta decision
                    assert v["median_cp"] == -1  # PValuePacket.getMetaDecision :212-218
                    dslots.setdefault(v["paxos_id"], []).append((v["slot"], v["request_id"]))
        for name, ss in dslots.items():  # every slot's decision is journaled once, in slot order, for the logged request
            assert [x[0] for x in ss] == list(range(1, len(ss) + 1))
            assert all(seen[rid][0] == name for _, rid in ss)
        assert journal.replay_decisions(d.j.files).keys() == dslots.keys()
        # every first request of every decided slot is in every replica's journal, byte-exact
        for rid, (name, val) in seen.items():
            assert sent[rid] == (name, val)
        for name, ss in slots.items():
            assert ss == list(range(1, len(ss) + 1))  # one logged ACCEPT per slot, in slot order
        assert d.accepts_written == sum(len(v) for v in slots.values()) == pm.num_decisions
        assert d.decisions_written == pm.num_decisions
        rec = journal.replay_accepts(d.j.files)
        assert set(rec) == set(slots) and all(len(rec[n]) == len(slots[n]) for n in rec)


def test_journal_roundtrip_cpu(oracle_lib, tmp_path):
    check(*run(oracle_lib, tmp_path))


def packets(drainer):
    return [p for f in drainer.j.files for p in journal.read_journal(f)]


def same_packets(drainers_a, drainers_b):
    """same packets in the same order on both (entry times differ: compare with entryTime masked)"""
    for a, b in zip(drainers_a, drainers_b):
        pa, pb = packets(a), packets(b)
        assert len(pa) == len(pb)
        for x, y in zip(pa, pb):
            vx, vy = journal.parse_packet(x), journal.parse_packet(y)
            assert vx["kind"] == vy["kind"]
            keys = (("paxos_id", "request_id", "slot", "bnum", "bcoord", "median_cp", "sender", "value", "n_batched")
                    if vx["kind"] == "ACCEPT" else ("paxos_id", "request_id", "slot", "bnum", "bcoord", "median_cp", "stop"))
            for k in keys:
                assert vx[k] == vy[k]


@pytest.mark.gpu
def test_journal_roundtrip_gpu(cuda_lib, oracle_lib, tmp_path):
    pm, dr, sent = run(cuda_lib, tmp_path / "gpu")
    check(pm, dr, sent)
    pm2, dr2, _ = run(oracle_lib, tmp_path / "cpu")
    same_packets(dr, dr2)


@pytest.mark.gpu
def test_journal_roundtrip_gpu_across_ring_wraps(cuda_lib, oracle_lib, tmp_path):
    """a 64 KiB ring, ~8 KB per lane and round: it wraps at least twice, and drains see the skips to the ring start"""
    ring = 1 << 16
    kw = dict(n_groups=30, rounds=24, log_ring_bytes=ring)
    pm, dr, sent = run(cuda_lib, tmp_path / "gpu", **kw)
    check(pm, dr, sent)
    assert all(pm.engine.log_head(l) > 2 * ring for l in range(3)), "the ring was sized to wrap twice"
    pm2, dr2, _ = run(oracle_lib, tmp_path / "cpu", **kw)
    same_packets(dr, dr2)


class RelaidRing:
    """log_head / log_read of one lane over a ring that an (unwrapped) oracle log was re-laid into the way the device
    lays it out (relay_into_small_ring)"""

    def __init__(self, ring, head, cap):
        self.cfg = types.SimpleNamespace(log_ring_bytes=cap)
        self.ring, self.head, self.cap = ring, head, cap

    def log_head(self, lane):
        return self.head

    def log_read(self, lane, start, nbytes):
        return self.ring.take(np.arange(start, start + nbytes) % self.cap)


def test_drain_across_ring_wraps_journals_every_segment(oracle_lib, tmp_path):
    """Drained once per call from a ring that wraps, the journal equals the one drained from the unwrapped ring: the
    segments after a skip to the ring start are journaled, and stale segments in the skipped tail are not."""
    G = 40
    eng = Engine(oracle_lib, make_config(oracle_lib, max_groups=G, max_batch_recs=4096, max_batch_payload=1 << 20))
    eng.create_groups(group_descs(G))
    rng = np.random.default_rng(6)
    heads = [0]
    for r in range(12):
        sel = np.arange(G)[rng.random(G) < 0.8]
        reqs, pay = make_requests(np.repeat(sel, np.where(rng.random(len(sel)) < 0.2, 2, 1)), payload_len=3 + r,
                                  seed=6, round_no=r)
        eng.round(reqs, pay)
        heads.append(eng.log_head(0))

    def lookup(gid, rid):
        return f"NoopPaxosApp{gid}", 0, NODES[0], 0

    want = journal.LogDrainer(eng, 0, journal.Journaler(str(tmp_path / "flat") + "/", NODES[0]), lookup)
    want.drain()
    want.j.close()
    buf = eng.log_read(0)
    cap = 1 << int(np.ceil(np.log2(2.2 * max(b - a for a, b in zip(heads[:-1], heads[1:])))))
    got = journal.LogDrainer(None, 0, journal.Journaler(str(tmp_path / "ring") + "/", NODES[0]), lookup)
    for k in range(2, len(heads) + 1):  # the ring as it is after each call
        ring, head, _, _ = relay_into_small_ring(buf, heads[:k], cap)
        got.engine = RelaidRing(ring, head, cap)
        got.drain()
    got.j.close()
    assert head > 2 * cap, "the ring wraps more than twice"
    assert got.accepts_written == want.accepts_written > 0
    assert got.decisions_written == want.decisions_written > 0
    assert packets(got) == packets(want)
    eng.close()
