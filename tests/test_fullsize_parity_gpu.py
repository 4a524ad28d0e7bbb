"""GPU-vs-oracle parity at BASELINE.json's FULL sizes (VERDICT r1 item 2): 2,500..25,000-block grids, a log-ring
wrap inside the run, 32-bit plane indices near their limits -- what the small parity tests cannot reach.

  cfg2      100 K groups x 3 replicas x 1 B, 8 rounds, the log ring wraps inside the run
  1 M       1 M groups x 3 replicas x 1 B, 3 rounds
  cfg3      125 K groups (the per-GPU shard of 1 M groups over 8 GPUs) x 64 B, 3 rounds
  cfg5      10 M groups created on the device, 1 % of them active in a round, checked against the oracle holding the
            active subset (oracle gid k <-> device gid active[k])

Everything is compared bit for bit (integer / byte work): request status, EXEC records per lane, every state row,
every counter, every log image and logged payload byte (per round, through the ring).  The criterion is the
reference's own: identical, gap-free, in-order execution on every replica (testing/TESTPaxosApp.java:179-213).
"""
import numpy as np
import pytest

from helpers import Engine, abi, canon, exec_by_lane, group_descs_fast, make_config, make_requests_fast

pytestmark = pytest.mark.gpu


def read_new_log(e, lane, prev_head, ring_cap=None):
    """segments appended since prev_head: [(hdr, images, payload)], new head"""
    head = e.log_head(lane)
    buf = e.log_read(lane, prev_head, head - prev_head)
    return [(h, i, p) for (h, i, p, _) in abi.parse_log(buf, ring_cap, prev_head)], head


def compare_round_logs(eo, eg, heads_o, heads_g, n_lanes, ring_cap):
    for l in range(n_lanes):
        so, heads_o[l] = read_new_log(eo, l, heads_o[l])
        sg, heads_g[l] = read_new_log(eg, l, heads_g[l], ring_cap)
        assert len(so) == len(sg) > 0, (l, len(so), len(sg))
        for (ho, io_, po), (hg, ig, pg) in zip(so, sg):
            for f in ("type", "lane", "payload_bytes", "seq", "rec_bytes", "n_slots"):
                assert int(ho[f]) == int(hg[f]), f"lane {l} seg hdr {f}"
            co, cg = canon(io_), canon(ig)
            assert len(co) == len(cg)
            for f in co.dtype.names:
                if f != "payload_off":
                    assert np.array_equal(co[f], cg[f]), f"lane {l} log image field {f}"
            if int(ho["rec_bytes"]) == 48 and len(co):  # logged payload bytes, vectorised for equal lengths
                ln = co["payload_len"].astype(np.int64)
                if np.all(ln == ln[0]):
                    L0 = int(ln[0])
                    ao = co["payload_off"].astype(np.int64)[:, None] + np.arange(L0)[None, :]
                    bo = cg["payload_off"].astype(np.int64)[:, None] + np.arange(L0)[None, :]
                    assert np.array_equal(po[ao], pg[bo]), f"lane {l} logged payload bytes"
                else:
                    for a, b in zip(co, cg):
                        x, y, n = int(a["payload_off"]), int(b["payload_off"]), int(a["payload_len"])
                        assert np.array_equal(po[x: x + n], pg[y: y + n])


def compare_rows(eo, eg, gids_o, gids_g, n_lanes, skip=("gid",)):
    for l in range(n_lanes):
        ro, rg = eo.dump_rows(gids_o, l), eg.dump_rows(gids_g, l)
        for f in ro.dtype.names:
            if f not in skip:
                assert np.array_equal(ro[f], rg[f]), f"lane {l} row field {f}"


def run_parity(oracle_lib, cuda_lib, G, P, rounds, ring_bytes, mode="round", check_wrap=False):
    R = 3
    pay_stride = ((P + 15) // 16) * 16
    kw = dict(max_groups=G, max_batch_recs=G, max_batch_payload=G * pay_stride + 16, log_ring_bytes=ring_bytes)
    eo, eg = Engine(oracle_lib, make_config(oracle_lib, **kw)), Engine(cuda_lib, make_config(cuda_lib, **kw))
    d = group_descs_fast(G)
    eo.create_groups(d)
    eg.create_groups(d)
    gids = np.arange(G)
    heads_o, heads_g = [0] * R, [0] * R
    wrapped = False
    for r in range(rounds):
        reqs, pay = make_requests_fast(gids, payload_len=P, seed=3, round_no=r, entry_lane=r % R)
        so, xo, extra_o = getattr(eo, mode)(reqs, pay)
        sg, xg, extra_g = getattr(eg, mode)(reqs, pay)
        assert np.array_equal(so, sg), f"round {r} status"
        assert len(extra_o) == len(extra_g) == 0
        h0 = heads_g[0]
        compare_round_logs(eo, eg, heads_o, heads_g, R, ring_bytes)
        now_wrapped = heads_g[0] // ring_bytes > h0 // ring_bytes or heads_g[0] > ring_bytes
        for l, (a, b) in enumerate(zip(exec_by_lane(xo, R), exec_by_lane(xg, R))):
            assert len(a) == len(b) == G, f"round {r} lane {l}"
            for f in a.dtype.names:
                # payload_off = ring position / 16 of the logged blob: the oracle's log is unbounded, so positions
                # agree only until the device ring has wrapped (then the bytes behind them are checked instead)
                if f != "payload_off" or not now_wrapped:
                    assert np.array_equal(a[f], b[f]), f"round {r} lane {l} exec {f}"
            assert np.all(b["slot"] == r + 1), "in-order, gap-free"
        if now_wrapped and not wrapped:  # the EXEC records of the round that wrapped point at the request bytes
            ex = exec_by_lane(xg, R)[0]
            ring = eg.log_read(0, max(heads_g[0] - ring_bytes, 0), min(heads_g[0], ring_bytes))
            base = max(heads_g[0] - ring_bytes, 0)
            sel = np.arange(0, G, max(G // 997, 1))
            for k in sel:
                pos = int(ex["payload_off"][k]) * 16
                ab = (heads_g[0] // ring_bytes) * ring_bytes + pos
                if ab >= heads_g[0]:
                    ab -= ring_bytes
                want = pay[int(reqs["payload_off"][ex["gid"][k]]): int(reqs["payload_off"][ex["gid"][k]]) + P]
                assert np.array_equal(ring[ab - base: ab - base + P], want), "EXEC payload reference after the ring wrap"
        wrapped = wrapped or now_wrapped
    if check_wrap:
        assert wrapped, "the run was sized to wrap the log ring"
    compare_rows(eo, eg, gids, gids, R, skip=())
    co, cg = eo.counters(), eg.counters()
    co.pop("kernel_launches"), cg.pop("kernel_launches")
    assert co == cg
    assert co["decisions_made"] == G * rounds and co["executed"] == R * G * rounds
    eo.close()
    eg.close()


@pytest.mark.parametrize("mode", ["round", "round_phases"])
def test_fullsize_cfg2_100k_groups_with_ring_wrap(oracle_lib, cuda_lib, mode):
    # one round appends ~11 MB per lane: a 64 MiB ring wraps in round 6 of 8
    run_parity(oracle_lib, cuda_lib, G=100_000, P=1, rounds=8, ring_bytes=1 << 26, mode=mode, check_wrap=True)


def test_fullsize_1m_groups(oracle_lib, cuda_lib):
    run_parity(oracle_lib, cuda_lib, G=1_000_000, P=1, rounds=3, ring_bytes=1 << 29)


def test_fullsize_cfg3_shard_125k_groups_64_bytes(oracle_lib, cuda_lib):
    run_parity(oracle_lib, cuda_lib, G=125_000, P=64, rounds=3, ring_bytes=1 << 27)


def test_fullsize_cfg5_10m_groups_one_percent_active(oracle_lib, cuda_lib):
    """10 M groups resident on the device (compact idle state: PaxosInstanceStateMachine.java:91-114 is why gigapaxos
    scales in groups); each round a 1 % subset is active, some groups with several requests (one batched slot)."""
    GT, R = 10_000_000, 3
    rng = np.random.default_rng(11)
    active = np.sort(rng.choice(GT, size=GT // 100, replace=False)).astype(np.uint32)
    A = len(active)
    eg = Engine(cuda_lib, make_config(cuda_lib, max_groups=GT, max_batch_recs=4 * A, max_batch_payload=64 * A,
                                      log_ring_bytes=1 << 28))
    for lo in range(0, GT, 2_000_000):  # batch creation, 2 M groups per call (PaxosManager.java:664-691)
        eg.create_groups(group_descs_fast(2_000_000, gid0=lo, name0=lo))
    eo = Engine(oracle_lib, make_config(oracle_lib, max_groups=A, max_batch_recs=4 * A, max_batch_payload=64 * A,
                                        log_ring_bytes=1 << 28))
    do = group_descs_fast(A)
    from helpers import java_hash_numbered
    do["name_hash"] = java_hash_numbered("NoopPaxosApp", active.astype(np.int64))
    eo.create_groups(do)
    compare_rows(eo, eg, np.arange(A), active, R)
    for r, b in enumerate([1, 1, 4]):  # requests per active group: 1, 1, then 4 (a batched slot per group)
        sub = np.arange(A) if b == 1 else np.arange(0, A, 3)
        idx_o = np.repeat(sub, b)
        reqs_o, pay = make_requests_fast(idx_o, payload_len=1, seed=8, round_no=r, entry_lane=r % R)
        reqs_g = reqs_o.copy()
        reqs_g["gid"] = active[idx_o]
        so, xo, extra_o = eo.round(reqs_o, pay)
        sg, xg, extra_g = eg.round(reqs_g, pay)
        assert np.array_equal(so, sg)
        assert len(extra_o) == len(extra_g) == 0
        for a, c in zip(exec_by_lane(xo, R), exec_by_lane(xg, R)):
            assert len(a) == len(c) == len(sub)
            assert np.array_equal(active[a["gid"]], c["gid"])
            for f in ("slot", "req_id", "flags"):
                assert np.array_equal(a[f], c[f]), f
            assert np.all((c["flags"] >> 16) == b)
    compare_rows(eo, eg, np.arange(A), active, R)
    # idle groups were not touched
    idle = np.setdiff1d(np.arange(0, GT, 9973, dtype=np.uint32), active)
    rows = eg.dump_rows(idle, 0)
    assert np.all(rows["acc_slot"] == 1) and np.all(rows["state"] == abi.ST_ACTIVE_1)
    co, cg = eo.counters(), eg.counters()
    co.pop("kernel_launches"), cg.pop("kernel_launches")
    assert co == cg
    eo.close()
    eg.close()
