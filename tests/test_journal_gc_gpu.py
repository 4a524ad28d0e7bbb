"""H100: journal garbage collection on the device (gpx_journal_compact_device through the C ABI, journal.JournalCompactor)
against journal.compact_files + apply_compaction on the same journal.  A PaxosManager with 3 lanes journals through
DeviceLogDrainer with a small file size (many rolls) and a small checkpoint interval; each lane's directory is copied,
one copy is collected on the device and the other on the host, and the two directories are byte-identical after the
merges -- with a view change's PREPAREs.  A 100 K-group round's frames, rolled into files, compact as compact_files
does.  Malformed frames are GPX_EINVAL with their indices listed."""
import os
import shutil

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


def journaled_manager(lib, tmp_path, n_groups=12, rounds=24, max_log=3000):
    eng = Engine(lib, make_config(lib, max_groups=64, max_batch_recs=1024, max_batch_payload=1 << 18,
                                  checkpoint_interval=4))
    pm = PaxosManager(eng, [NoopPaxosApp() for _ in NODES], NODES)
    names = [f"NoopPaxosApp{i}" for i in range(n_groups)]
    pm.createPaxosInstanceBatch({n: None for n in names}, NODES)
    wire.set_group_names(eng, [pm.instances[n].gid for n in names], names)
    known = {}

    def meta_source(miss):
        return meta_records([(g, r) + known[(g, r)] for g, r in zip(miss["gid"].tolist(), miss["req_id"].tolist())])

    dev = [journal.DeviceLogDrainer(eng, l, journal.Journaler(str(tmp_path / "j") + "/", NODES[l], max_log),
                                    meta_source) for l in range(3)]
    rng = np.random.default_rng(5)

    def step():
        pm.run_round()
        for d in dev:
            d.drain()
    for r in range(rounds):
        for n in names:
            for _ in range(int(rng.integers(1, 4))):
                rid = pm.propose(n, bytes(rng.integers(97, 123, size=int(rng.integers(1, 20))).astype(np.uint8)),
                                 entry_node=NODES[int(rng.integers(0, 3))])
                req = pm.outstanding[rid]
                known[(pm.instances[n].gid, rid)] = (req.entry_replica, int(req.entry_time * 1000))
        step()
        if r == rounds // 2:  # the next node takes over every group: logged PREPAREs
            for c in range(3):
                assert all(pm.runForCoordinators(names[c::3], (c + 1) % 3).values())
            step()
    return pm, dev


def gc_slot_of(pm, gc):
    def f(pid, ver):
        inst = pm.instances.get(pid)
        return None if inst is None or inst.version != ver else int(gc[inst.gid])
    return f


def dir_bytes(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


def test_device_gc_equals_compact_files(cuda_lib, tmp_path):
    pm, dev = journaled_manager(cuda_lib, tmp_path)
    assert len(pm.checkpoints) > 0
    total_dropped = 0
    for lane, d in enumerate(dev):
        j = d.j
        assert len(j.files) > 6
        gc = pm.journal_gc_slots(lane)
        assert (gc > 0).sum() > 0
        # the host copy: the same directory, compacted by the model
        host_dir = str(tmp_path / f"host{lane}")
        shutil.copytree(j.dir, host_dir)
        hj = journal.Journaler.__new__(journal.Journaler)
        hj.dir, hj.max, hj.cur = host_dir, j.max, os.path.join(host_dir, os.path.basename(j.cur))
        hj.files = [os.path.join(host_dir, os.path.basename(f)) for f in j.files]
        files = [f for f in hj.files if f != hj.cur]
        want = journal.compact_files(files + [hj.cur], gc_slot_of(pm, gc))[:-1]
        journal.apply_compaction(hj, files, want)
        got = journal.JournalCompactor(pm.engine, j).compact(gc)
        assert got == want
        assert dir_bytes(j.dir) == dir_bytes(host_dir)
        assert [os.path.basename(f) for f in j.files] == [os.path.basename(f) for f in hj.files]
        assert len(j.files) < len(files) + 1  # something was deleted or merged
        total_dropped += sum(r.dropped for r in got)
        kinds = {journal.parse_packet(p)["kind"] for f in j.files for p in journal.read_journal(f)}
        assert {"ACCEPT", "DECISION"} <= kinds
    assert total_dropped > 100
    for d in dev:
        d.j.close()
    pm.engine.close()


def test_a_100k_group_round(cuda_lib, tmp_path):
    import torch
    G = 100_000
    eng = Engine(cuda_lib, make_config(cuda_lib, max_groups=G, max_batch_recs=2 * G, max_batch_payload=64 << 20))
    eng.create_groups(group_descs_fast(G))
    gids = np.arange(G, dtype=np.uint32)
    wire.set_group_names(eng, gids, [f"NoopPaxosApp{i}" for i in range(G)])
    blobs = []
    for r in range(2):
        reqs, pay = make_requests_fast(gids, payload_len=16, seed=3 + r)
        eng.round(reqs, pay)
        meta = np.zeros(G, abi.journal_req_dtype)
        meta["gid"], meta["req_id"], meta["entry_node"] = reqs["gid"], reqs["req_id"], reqs["entry_node"]
        meta["entry_time"] = 1760000000000 + np.arange(G)
        meta = meta[np.lexsort((meta["req_id"], meta["gid"]))]
        dmeta = torch.from_numpy(meta.view(np.uint8).reshape(-1, 24).copy()).cuda()
        f = eng.log_frame_device(0, 0 if r == 0 else eng_from, dmeta, len(meta))
        assert f.rc == 0
        eng_from = f.from_
        eng.log_release(0, f.from_)
        data = f.frames.cpu().numpy().tobytes()
        half = eng.L.journal_index(data)[len(eng.L.journal_index(data)) // 2]
        blobs += [data[:half], data[half:]]
    rows = eng.dump_rows(gids, 0)
    rng = np.random.default_rng(1)
    slots = rows["acc_slot"].astype(np.int64)
    gc = np.where(rng.random(G) < 0.5, slots - 1, -1).astype(np.int32)  # about half the groups drop their frames
    paths = []
    for i, b in enumerate(blobs):
        p = tmp_path / f"f{i}"
        p.write_bytes(b)
        paths.append(str(p))
    names = {f"NoopPaxosApp{i}": i for i in range(G)}
    want = journal.compact_files(paths, lambda pid, ver: int(gc[names[pid]]) if ver == 0 and pid in names else None,
                                 last_readonly=False)
    file_off = np.zeros(len(blobs) + 1, np.uint32)
    file_off[1:] = np.cumsum([len(b) for b in blobs])
    starts = np.concatenate([eng.L.journal_index(b, int(o)) for b, o in zip(blobs, file_off[:-1])])
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    r = eng.journal_compact_device(d(np.frombuffer(b"".join(blobs), np.uint8).copy()), int(file_off[-1]), d(file_off),
                                   d(starts), d(gc), False)
    assert r.rc == 0
    out = r.out.cpu().numpy()
    fr = r.files.cpu().numpy().reshape(-1).view(abi.journal_file_dtype)
    got = [journal.CompactedFile(int(x["status"]), out[int(x["out_off"]): int(x["out_off"]) + int(x["out_bytes"])]
                                 .tobytes() if int(x["status"]) == journal.JGC_COMPACTED else None, int(x["kept"]),
                                 int(x["dropped"]), int(x["unresolved"])) for x in fr]
    assert got == want
    dropped = sum(x.dropped for x in got)
    assert 0.3 < dropped / len(starts) < 0.7
    eng.close()


def test_errors_on_the_device(cuda_lib):
    import torch
    eng = Engine(cuda_lib, make_config(cuda_lib, max_groups=16, max_batch_recs=64, max_batch_payload=1 << 16))
    eng.create_groups(group_descs_fast(16))
    wire.set_group_names(eng, np.arange(16, dtype=np.uint32), [f"g{i}" for i in range(16)])
    good = wire.journal_frame(journal.decision_json("g1", 0, 5, 1, 100, -1, 9, 100, 7))
    bad = wire.journal_frame(b'{"type":90,"PT":6,"ID":"g1"}')
    data = good + bad + good
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    gc = d(np.full(16, -1, np.int32))
    off = d(np.array([0, len(data)], np.uint32))
    starts = eng.L.journal_index(data)
    r = eng.journal_compact_device(d(np.frombuffer(data, np.uint8).copy()), len(data), off, d(starts), gc, False)
    assert r.rc == abi.GPX_EINVAL and r.bad.cpu().numpy().tolist() == [1]
    starts[1] += 1  # a start that disagrees with the previous frame's length
    r = eng.journal_compact_device(d(np.frombuffer(data, np.uint8).copy()), len(data), off, d(starts), gc, False)
    assert r.rc == abi.GPX_EINVAL and 0 in r.bad.cpu().numpy().tolist()
    with pytest.raises(abi.GpxError):  # file_off past the bytes
        eng.journal_compact_device(d(np.frombuffer(data, np.uint8).copy()), len(data),
                                   d(np.array([0, len(data) + 4], np.uint32)), d(starts), gc, False)
    with pytest.raises(abi.GpxError):  # a GC slot per group
        eng.journal_compact_device(d(np.frombuffer(data, np.uint8).copy()), len(data), off, d(starts), gc[:4], False)
    eng.close()
