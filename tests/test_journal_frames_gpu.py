"""H100: journal frames written on the device (gpx_log_frame_device through the C ABI, journal.DeviceLogDrainer) against
journal.LogDrainer on the same engine.  A PaxosManager with 3 lanes journals every lane twice, once per drainer, into
two directories: the files are byte-identical, roll points included, and replay_accepts / replay_decisions agree --
with batched proposals entering at every node, a view change's logged PREPAREs, and across many ring wraps with
log_backpressure.  A 100 K-group round is framed on every lane and checked against LogDrainer on one lane."""
import numpy as np
import pytest

from gigapaxos_b200 import journal, wire
from gigapaxos_b200.paxos_manager import NoopPaxosApp, PaxosManager
from helpers import Engine, abi, group_descs_fast, make_config, make_requests_fast

pytestmark = pytest.mark.gpu
NODES = [100, 101, 102]


def meta_records(rows):
    m = np.zeros(len(rows), abi.journal_req_dtype)
    if rows:
        m["gid"], m["req_id"], m["entry_node"], m["entry_time"] = (np.array(c) for c in zip(*rows))
    return m


def run(lib, tmp_path, n_groups=6, rounds=6, view_change=True, max_log=2000, **cfg):
    eng = Engine(lib, make_config(lib, max_groups=64, max_batch_recs=1024, max_batch_payload=1 << 18, **cfg))
    pm = PaxosManager(eng, [NoopPaxosApp() for _ in NODES], NODES)
    names = [f"NoopPaxosApp{i}" for i in range(n_groups)]
    pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
    wire.set_group_names(eng, [pm.instances[n].gid for n in names], names)
    known = {}  # (gid, req_id) -> (paxosID, version, entryReplica, entryTime ms)

    def lookup(gid, rid):
        if rid == -1:
            return pm.gid_name[gid], 0, 0, 0
        return known[(gid, rid)]

    def meta_source(miss):
        return meta_records([(g, r, known[(g, r)][2], known[(g, r)][3]) for g, r in zip(miss["gid"].tolist(),
                                                                                          miss["req_id"].tolist())])

    host = [journal.LogDrainer(eng, l, journal.Journaler(str(tmp_path / "host") + "/", NODES[l], max_log), lookup)
            for l in range(3)]
    dev = [journal.DeviceLogDrainer(eng, l, journal.Journaler(str(tmp_path / "dev") + "/", NODES[l], max_log),
                                    meta_source) for l in range(3)]
    rng = np.random.default_rng(4)
    for r in range(rounds):
        fresh = []
        for n in names:
            for _ in range(int(rng.integers(1, 6))):
                val = bytes(rng.integers(97, 123, size=int(rng.integers(1, 30))).astype(np.uint8))
                rid = pm.propose(n, val, entry_node=NODES[int(rng.integers(0, 3))])
                req = pm.outstanding[rid]
                gid = pm.instances[n].gid
                known[(gid, rid)] = (n, 0, req.entry_replica, int(req.entry_time * 1000))
                fresh.append((gid, rid, req.entry_replica, int(req.entry_time * 1000)))
        if r % 2:  # half the rounds' requests are in the table ahead of the drain, the others come as misses
            for d in dev:
                d.add(meta_records(fresh))
        pm.run_round()
        for h, d in zip(host, dev):
            h.drain()
            d.drain()
    if view_change:  # the next node takes over every group: logged PREPAREs
        for c in range(3):
            won = pm.runForCoordinators(names[c::3], (c + 1) % 3)
            assert all(won.values())
        pm.run_round()
        for h, d in zip(host, dev):
            h.drain()
            d.drain()
    for d in host + dev:
        d.j.close()
    return pm, host, dev


def same_files(host, dev, want_prepare=False):
    kinds = set()
    for h, d in zip(host, dev):
        assert len(h.j.files) == len(d.j.files) > 1  # rolled at the same points
        total = 0
        for a, b in zip(h.j.files, d.j.files):
            with open(a, "rb") as x, open(b, "rb") as y:
                xa, yb = x.read(), y.read()
            assert xa == yb  # the file opened by the last roll may be empty in both
            total += len(xa)
            kinds |= {journal.parse_packet(p)["kind"] for p in journal.read_journal(a)}
        assert total > 0
        assert journal.replay_accepts(h.j.files) == journal.replay_accepts(d.j.files)
        assert journal.replay_decisions(h.j.files) == journal.replay_decisions(d.j.files)
        assert d.frames_written == h.accepts_written + h.decisions_written
    assert {"ACCEPT", "DECISION"} <= kinds
    if want_prepare:
        assert "PREPARE" in kinds


def test_device_frames_equal_log_drainer(cuda_lib, tmp_path):
    pm, host, dev = run(cuda_lib, tmp_path)
    same_files(host, dev, want_prepare=True)
    pm.engine.close()


def test_device_frames_across_ring_wraps_with_backpressure(cuda_lib, tmp_path):
    """a 64 KiB ring with log_backpressure: the device drainer releases what it framed, the ring wraps 8 times"""
    ring = 1 << 16
    pm, host, dev = run(cuda_lib, tmp_path, n_groups=30, rounds=40, view_change=False, max_log=20000,
                        log_ring_bytes=ring, log_backpressure=1)
    assert all(pm.engine.log_head(l) > 8 * ring for l in range(3)), "the ring was sized to wrap 8 times"
    same_files(host, dev)
    pm.engine.close()


def test_a_100k_group_round(cuda_lib, tmp_path):
    import torch
    G = 100_000
    eng = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, max_batch_recs=2 * G, max_batch_payload=64 << 20))
    eng.create_groups(group_descs_fast(G))
    gids = np.arange(G, dtype=np.uint32)
    wire.set_group_names(eng, gids, [f"NoopPaxosApp{i}" for i in range(G)])
    reqs, pay = make_requests_fast(gids, payload_len=16, seed=3)
    eng.round(reqs, pay)
    meta = np.zeros(G, abi.journal_req_dtype)
    meta["gid"], meta["req_id"], meta["entry_node"] = reqs["gid"], reqs["req_id"], reqs["entry_node"]
    meta["entry_time"] = 1760000000000 + np.arange(G)
    meta = meta[np.lexsort((meta["req_id"], meta["gid"]))]
    t = {(int(m["gid"]), int(m["req_id"])): (int(m["entry_node"]), int(m["entry_time"])) for m in meta}
    dmeta = torch.from_numpy(meta.view(np.uint8).reshape(-1, 24).copy()).cuda()
    for lane in range(3):
        r = eng.log_frame_device(lane, 0, dmeta, len(meta))
        assert r.rc == 0 and r.from_ == eng.log_head(lane) and r.sizes[1] == 2 * G
        got = r.frames.cpu().numpy().tobytes()
        if lane == 0:  # LogDrainer, one interpreted call per image, is the slow reference: one lane of the round
            class Collect:
                buf = bytearray()

                def append(self, p):
                    self.buf += wire.journal_frame(p)

                def end_batch(self):
                    pass
            d = journal.LogDrainer(eng, 0, Collect(), lambda g, q: (f"NoopPaxosApp{g}", 0) + t[(g, q)])
            d.drain()
            assert got == bytes(d.j.buf)
        else:  # the others: a sample of frames parsed back against the table
            path = tmp_path / f"l{lane}"
            path.write_bytes(got)
            pkts = list(journal.read_journal(str(path)))
            assert len(pkts) == 2 * G
            for p in pkts[:: 997]:
                v = journal.parse_packet(p)
                gid = int(v["paxos_id"][len("NoopPaxosApp"):])
                assert (v["entry_replica"], v["entry_time"]) == t[(gid, v["request_id"])]
        eng.log_release(lane, r.from_)
    eng.close()
