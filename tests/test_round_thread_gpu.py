"""GPU parity of the two in-order round kernels: k_round_g (one thread per group, the default for n_lanes <= 3) against
k_round (a team of n_lanes threads per group, forced with gpx_set_round_mode 3 / 4).

Two engines in the same state run the same rounds, one per kernel, and everything they produce is compared byte for
byte: status, EXEC rows (around a caller buffer at 8 mod 16 as well as at 0 mod 16), compact summaries, every lane's
log ring from its start to its head, the rows of every group and the counters.  The rounds mix the in-order case with
groups the slow kernel takes over inside the same warps: STOPs, groups with a remote member (a non-local or absent
coordinator), stopped groups, and -- driven by the adversarial schedule generator -- batched runs, outstanding
proposals, occupied window entries and NACKed ballots.
"""
import ctypes as C

import numpy as np
import pytest

from fuzz import Fuzzer
from helpers import Engine, abi, group_descs, make_config, make_requests
from test_round_parity_gpu import compare_logs
from wrap_cases import BALLOT_BASE, NODES, SLOT_BASES, shift_rows

pytestmark = pytest.mark.gpu

TEAM = 3       # gpx_set_round_mode: the team kernel, device tail launch of k_round_slow
TEAM_HOST = 4  # the team kernel, host-launched k_round_slow
THREAD_HOST = 2
REMOTE = 900   # a member node with no lane in the engine
LENS = np.array([0, 1, 15, 16, 17, 100], dtype=np.uint32)
NODEF = dict(gc_majority_executed=0, log_meta_decisions=0, journaling_enabled=0, checkpoint_interval=3)


def set_mode(e, mode):
    e.L.check(e.L.fn("set_round_mode")(e.handle, C.c_int(mode)))


def engines(cuda_lib, L, G, base, **kw):
    """(thread-kernel engine, team-kernel engine): G - G // 5 groups whose members are the L lanes, then G // 5 groups
    with one more, remote member; every slot and ballot moved to start at `base` / BALLOT_BASE when base is not None"""
    cfg = dict(max_groups=G, n_lanes=L, lane_node=NODES[:L], window=8, max_group_size=L + 1, max_batch_recs=1 << 14,
               max_batch_payload=1 << 21, log_ring_bytes=1 << 24, checkpoint_interval=4)
    cfg.update(kw)
    es = [Engine(cuda_lib, make_config(cuda_lib, **cfg)) for _ in range(2)]
    set_mode(es[1], TEAM)
    n_rem = G // 5
    for e in es:
        e.create_groups(group_descs(G - n_rem, members=NODES[:L]))
        e.create_groups(group_descs(n_rem, members=NODES[:L] + [REMOTE], gid0=G - n_rem, prefix="RemoteApp"))
    if base is not None:
        gids = np.arange(G)
        rows = np.concatenate([es[0].dump_rows(gids, l) for l in range(L)])
        rows = shift_rows(rows, base - int(rows["acc_slot"][0]), BALLOT_BASE)
        for e in es:
            e.load_rows(rows)
    return es


def requests(G, L, rng, r, aligned):
    """one request per present group (about one in eight absent), payload lengths from LENS, a STOP now and then;
    payloads 16-byte aligned in the arena, or back to back from an odd offset"""
    gids = np.nonzero(rng.random(G) >= 0.125)[0]
    lens = LENS[rng.integers(0, len(LENS), size=len(gids))]
    stop = rng.random(len(gids)) < (0.01 if r >= 2 else 0.0)
    entry = r % L
    reqs, pay = make_requests(gids, payload_len=lens, seed=61, round_no=r, entry_lane=entry, entry_node=NODES[entry],
                              stop_mask=stop)
    if not aligned:
        offs = (3 + np.concatenate([[0], np.cumsum(lens)[:-1]])).astype(np.uint32)
        body = np.zeros(3 + int(lens.sum()), dtype=np.uint8)
        for o, no, ln in zip(reqs["payload_off"], offs, lens):
            body[no: no + ln] = pay[o: o + ln]
        reqs["payload_off"], pay = offs, body
    return reqs, pay


def device_round(e, reqs, pay, exec_shift):
    """gpx_round_device with the EXEC rows at `exec_shift` bytes past a 512-byte aligned allocation pre-filled with a
    marker: -> (status, the whole EXEC allocation)"""
    import torch
    dev = torch.device("cuda", 0)
    n, L = len(reqs), e.n_lanes
    d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).to(dev)
    d_pay = torch.from_numpy(np.concatenate([pay, np.zeros(16, np.uint8)])).to(dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    d_exec = torch.full((n * L * 24 + 32,), 0xA5, dtype=torch.uint8, device=dev)
    bufs = abi.DevRoundBufs(d_reqs.data_ptr(), d_pay.data_ptr(), len(pay), n, d_status.data_ptr(),
                            d_exec.data_ptr() + exec_shift)
    torch.cuda.synchronize()
    e.L.check(e.L.fn("round_device")(e.handle, C.byref(bufs), None))
    torch.cuda.synchronize()
    return d_status.cpu().numpy(), d_exec.cpu().numpy()


def same_state(a, b, G, L):
    gids = np.arange(G)
    for l in range(L):
        ra, rb = a.dump_rows(gids, l), b.dump_rows(gids, l)
        assert ra.tobytes() == rb.tobytes(), f"rows of lane {l}"
    ca, cb = a.counters(), b.counters()
    ca.pop("kernel_launches"), cb.pop("kernel_launches")
    assert ca == cb, {k: (ca[k], cb[k]) for k in ca if ca[k] != cb[k]}
    return ca


def same_rings(a, b, L):
    for l in range(L):
        assert a.log_head(l) == b.log_head(l), f"lane {l} ring head"
        ra, rb = a.log_read(l), b.log_read(l)
        assert len(ra) > 0 and ra.tobytes() == rb.tobytes(), f"lane {l} ring bytes differ at {np.nonzero(ra != rb)[0][:8]}"


@pytest.mark.parametrize("L,conf,base", [(1, "def", None), (2, "def", None), (3, "def", None), (2, "nodef", None),
                                         (3, "nodef", None), (3, "def", "intmax"), (3, "def", "rs_codes"),
                                         (1, "nodef", "intmax")])
def test_device_rounds_byte_identical(cuda_lib, L, conf, base):
    """one request per group: every output of both kernels, byte for byte, the EXEC rows alternately at 0 and 8 mod
    16 and the payloads alternately aligned and at odd offsets"""
    G = 3001  # the last warp of the grid is partial
    a, b = engines(cuda_lib, L, G, None if base is None else SLOT_BASES[base], **(NODEF if conf == "nodef" else {}))
    rng = np.random.default_rng(L * 100 + len(conf))
    for r in range(8):
        reqs, pay = requests(G, L, rng, r, aligned=r % 2 == 0)
        shift = 8 if r % 4 < 2 else 0
        sa, xa = device_round(a, reqs, pay, shift)
        sb, xb = device_round(b, reqs, pay, shift)
        assert np.array_equal(sa, sb), f"round {r}: status differs at {np.nonzero(sa != sb)[0][:8]}"
        assert xa.tobytes() == xb.tobytes(), f"round {r}: EXEC bytes differ at {np.nonzero(xa != xb)[0][:8]}"
    c = same_state(a, b, G, L)
    same_rings(a, b, L)
    assert c["stops_executed"] > 0 and c["decisions_made"] > 4 * G
    for e in (a, b):
        e.close()


def extra_set(ex):
    """the extra queue's records as a sorted byte set; the log position of a BATCHED slot's blob (payload_off of a
    record with nreq > 1) depends on the order in which the slow kernel's blocks reserved space, so it is masked"""
    ex = ex.copy()
    ex["payload_off"][(ex["flags"] >> 16) > 1] = 0
    return np.sort(ex.view(np.uint8).reshape(len(ex), -1).view("V24").ravel())


@pytest.mark.parametrize("L", [1, 2, 3])
def test_compact_rounds_identical(cuda_lib, L):
    """compact output mode through the pipelined API: summaries byte for byte, the extra queue as a set (its order is
    the order in which the slow kernel's threads reached it)"""
    G = 2000
    a, b = engines(cuda_lib, L, G, None)
    rng = np.random.default_rng(7 + L)
    for r in range(6):
        counts = rng.choice([0, 1, 1, 1, 1, 1, 2, 4], size=G)
        gids = np.repeat(np.arange(G), counts)
        lens = LENS[rng.integers(0, len(LENS), size=len(gids))]
        stop = rng.random(len(gids)) < (0.01 if r >= 2 else 0.0)
        reqs, pay = make_requests(gids, payload_len=lens, seed=67, round_no=r, entry_lane=r % L,
                                  entry_node=NODES[r % L], stop_mask=stop)
        cap = 4 * len(reqs) * L + 64
        ra = a.round_wait(a.round_submit(reqs, pay, compact=True, extra_cap=cap))
        rb = b.round_wait(b.round_submit(reqs, pay, compact=True, extra_cap=cap))
        assert ra["sum"].tobytes() == rb["sum"].tobytes(), f"round {r}: summaries"
        assert ra["n_extra"] == rb["n_extra"]
        ea, eb = extra_set(ra["extra"]), extra_set(rb["extra"])
        assert ea.tobytes() == eb.tobytes(), f"round {r}: extra queue"
    same_state(a, b, G, L)
    compare_logs(a, b, L)
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("seed,R,modes", [(81, 1, (0, TEAM)), (82, 2, (0, TEAM)), (83, 3, (0, TEAM)),
                                          (84, 3, (THREAD_HOST, TEAM_HOST))])
def test_adversarial_schedules_agree(cuda_lib, seed, R, modes):
    """fused rounds in the states adversarial schedules leave behind (batched runs, outstanding proposals, occupied
    window entries, NACKs, coordinator changes), with the thread kernel in one engine and the team kernel in the other:
    outputs, rows, counters and ring heads after every few steps, the log images at the end"""
    f = Fuzzer([cuda_lib, cuda_lib], G=200, R=R, W=4, seed=seed)
    for e, m in zip(f.engines, modes):
        set_mode(e, m)
    decided = f.run(steps=50, check_every=5, fused_prob=0.3, round_prob=0.6)
    assert decided > 100
    compare_logs(f.engines[0], f.engines[1], R)
    f.close()


def test_round_mode_range(cuda_lib):
    e = Engine(cuda_lib, make_config(cuda_lib, max_groups=8))
    for m in range(5):
        set_mode(e, m)
    with pytest.raises(abi.GpxError):
        set_mode(e, 5)
    e.close()
