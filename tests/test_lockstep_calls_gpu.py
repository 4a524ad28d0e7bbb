"""GPU tests of every call that touches group state while k_round_g's lockstep records are VALID.

After a compacting round a group whose lanes advance in lockstep lives in its 32-byte record (gpx_dev.cuh, ls_rec),
and its acc_row, coord_row[cl] and ns_u[cl] words are at least one slot behind.  Every other launch that reads or
writes group state must come after ls_settle (gpx_engine.cu).  A missing settle does not crash: the call answers from
an old slot, or the next settle writes the old record over what the call wrote.

Twin engines run the same calls: one with k_round_g (compacts), one with the team kernel (never does).  Each case runs
two one-launch compacting rounds, the call under test with inputs chosen so that a stale plane changes the answer
(the call's groups hold VALID records), compares every output byte for byte, runs more compacting rounds and compares
rows, counters, log rings and log images.  The mixed-layout fuzz runs identity groups, which compact, beside groups
of lane subsets, permuted and remote members, against the CPU oracle and against the team twin.
"""
import ctypes as C
from collections import namedtuple

import numpy as np
import pytest

from fuzz import Fuzzer
from helpers import Engine, abi, exec_by_lane, group_descs, group_names, make_config, make_requests
from test_node_slots_compact_gpu import plain_requests, run_round, twins
from test_round_lockstep_gpu import compact_rounds
from test_round_parity_gpu import compare_logs
from test_round_thread_gpu import REMOTE, TEAM, THREAD_HOST, engines, same_rings, same_state, set_mode
from test_wire_device_gpu import DevNode
from wrap_cases import NODES, SLOT_BASES

from gigapaxos_b200 import wire

pytestmark = pytest.mark.gpu

G = 3001
DevIn = namedtuple("DevIn", "accepts blob sizes")  # what DevNode.accepts reads of a decoder's output


def as_set(recs):
    """records as a sorted byte set: where a kernel appends through an atomic counter, the order is its threads'"""
    recs = np.ascontiguousarray(recs)
    if len(recs) == 0:
        return b""
    return np.sort(recs.view(np.uint8).reshape(len(recs), -1).view(f"V{recs.dtype.itemsize}").ravel()).tobytes()


def wrap32(x):
    return ((np.asarray(x, dtype=np.int64) + 2**31) % 2**32 - 2**31).astype(np.int32)


def coord_view(e, gids, L):
    """per gid: (coordinator lane, that lane's row) -- read from the team twin, whose dump settles nothing"""
    rows = [e.dump_rows(gids, l) for l in range(L)]
    cl = np.full(len(gids), -1)
    for l in range(L):
        cl[rows[l]["coord_exists"] != 0] = l
    assert (cl >= 0).all(), "every identity group has a coordinator at a lane"
    return cl, np.choose(cl, rows)


def both(a, b, fn, what):
    """fn on both engines; outputs equal byte for byte"""
    oa, ob = fn(a), fn(b)
    for i, (x, y) in enumerate(zip(oa if isinstance(oa, tuple) else (oa,), ob if isinstance(ob, tuple) else (ob,))):
        xb = x if isinstance(x, bytes) else np.ascontiguousarray(x).tobytes()
        yb = y if isinstance(y, bytes) else np.ascontiguousarray(y).tobytes()
        assert xb == yb, f"{what}: output {i} differs"
    return oa


def oracle_twin(oracle_lib, a, L, base):
    """a CPU oracle engine in the state the twins start in (their config, every row of every lane)"""
    eo = Engine(oracle_lib, make_config(oracle_lib, max_groups=G, n_lanes=L, lane_node=NODES[:L], window=8,
                                        max_group_size=L + 1, max_batch_recs=1 << 14, max_batch_payload=1 << 21,
                                        checkpoint_interval=4))
    eo.create_groups(group_descs(G, members=NODES[:L]))
    if base is not None:
        eo.load_rows(np.concatenate([a.dump_rows(np.arange(G), l) for l in range(L)]))
    return eo


def trio_round(a, b, eo, L, r, reqs_pay=None):
    """one round (gpx_round) on the twins and, if given, the oracle: the twins byte for byte (the log position of a
    BATCHED slot's blob aside), the oracle's status and decided (slot, request) sequence per lane"""
    reqs, pay = reqs_pay if reqs_pay is not None else plain_requests(G, L, r)
    cap = 4 * len(reqs) * L + 256
    outs = [e.round(reqs, pay, extra_cap=cap) for e in (a, b)]
    for x in outs:
        for ex in x[1:]:
            ex["payload_off"][(ex["flags"] >> 16) > 1] = 0
    assert outs[0][0].tobytes() == outs[1][0].tobytes(), f"round {r}: status"
    assert outs[0][1].tobytes() == outs[1][1].tobytes(), f"round {r}: EXEC rows"
    assert as_set(outs[0][2]) == as_set(outs[1][2]), f"round {r}: extra EXEC rows"
    if eo is not None:
        so, xo, _ = eo.round(reqs, pay, extra_cap=cap)
        assert np.array_equal(outs[0][0], so), f"round {r}: status vs the oracle at {np.nonzero(outs[0][0] != so)[0][:8]}"
        for l, (x, y) in enumerate(zip(exec_by_lane(outs[0][1], L), exec_by_lane(xo, L))):
            for f in ("gid", "slot", "req_id", "flags"):
                bad = np.nonzero(x[f] != y[f])[0][:3] if len(x) == len(y) else [len(x), len(y)]
                assert len(x) == len(y) and not len(bad), f"round {r} lane {l} {f} vs the oracle: {bad} {x[bad[:1]]} {y[bad[:1]]}"
    return r + 1


def same_as_oracle(a, eo, L):
    for l in range(L):
        ra, ro = a.dump_rows(np.arange(G), l), eo.dump_rows(np.arange(G), l)
        for f in ra.dtype.names:
            assert np.array_equal(ra[f], ro[f]), f"lane {l} field {f} vs the oracle"
    ca, co = a.counters(), eo.counters()
    for k in ("decisions_made", "executed", "stops_executed", "preempted"):
        assert ca[k] == co[k], (k, ca[k], co[k])


# ---- the calls ---------------------------------------------------------------------------------------------------
def view_change(a, b, L, r, eo=None):
    """PREPAREs at a higher ballot from another lane's node for a strided subset (gpx_handle_prepares), one compacting
    round (the other groups' records are VALID again), then the elections (gpx_handle_prepare_replies): the prepared
    groups with their acceptors' replies, and a second subset whose replies come in as records -- as from the
    acceptors of a node that ran the PREPAREs itself -- while their records are VALID"""
    A = np.arange(1, G, 7, dtype=np.uint32)
    cl, row = coord_view(b, A, L)
    cand = (cl + 1) % L
    prep = np.zeros(len(A), dtype=abi.decision_dtype)
    prep["gid"], prep["slot"] = A, row["acc_slot"]
    prep["bnum"], prep["bcoord"] = wrap32(row["acc_bnum"].astype(np.int64) + 1), np.array(NODES)[cand]
    prep["flags"], prep["dst_mask"] = abi.F_PREPARE, (1 << L) - 1
    reps = both(a, b, lambda e: e.handle_prepares(prep), "prepare replies")
    assert eo.handle_prepares(prep).tobytes() == reps.tobytes(), "prepare replies vs the oracle"
    r = trio_round(a, b, eo, L, r)
    Cg = np.arange(4, G, 7, dtype=np.uint32)
    ccl, crow = coord_view(b, Cg, L)
    ccand = (ccl + 1) % L
    nb = wrap32(crow["acc_bnum"].astype(np.int64) + 1)
    fab = np.zeros(len(Cg) * L, dtype=abi.prepare_reply_dtype)
    fab["gid"] = np.repeat(Cg, L)
    fab["first_slot"] = np.repeat(wrap32(crow["acc_slot"].astype(np.int64) - 1), L)  # gcSlot: all before decided
    fab["bnum"], fab["bcoord"] = np.repeat(nb, L), np.repeat(np.array(NODES)[ccand], L)
    fab["who"] = [abi.who(m, int(c)) for c in ccand for m in range(L)]
    els = np.zeros(len(A) + len(Cg), dtype=abi.election_dtype)
    els["gid"] = np.concatenate([A, Cg])
    els["lane"] = np.concatenate([cand, ccand])
    els["bnum"] = np.concatenate([prep["bnum"], nb])
    els["bcoord"] = np.concatenate([prep["bcoord"], np.array(NODES)[ccand]])
    els["slot"] = np.concatenate([prep["slot"], crow["acc_slot"]])
    els["first_reply"] = np.arange(len(els)) * L
    els["n_replies"] = L
    allreps = np.concatenate([reps, fab])
    outs = both(a, b, lambda e: e.handle_prepare_replies(els, allreps), "election results")
    assert eo.handle_prepare_replies(els, allreps).tobytes() == outs.tobytes(), "election results vs the oracle"
    assert (outs["verdict"] == abi.EL_MAJORITY).all(), np.unique(outs["verdict"], return_counts=True)
    launches = []
    for _ in range(8):
        k0 = a.counters()["kernel_launches"]
        r = trio_round(a, b, eo, L, r)
        launches.append(a.counters()["kernel_launches"] - k0)
    assert launches[-2:] == [1, 1], f"the elected groups are back on the fast path: {launches}"
    same_as_oracle(a, eo, L)
    return r


def missing_decisions(a, b, L, r):
    """SYNC_DECISIONS fields of every group at every lane: the committed slot and the gap come from the acceptor
    slot, and a size_limit of 0 or 1 makes missing_too_much turn on it too"""
    gids = np.arange(G, dtype=np.uint32)
    for lane in range(L):
        for lim in (0, 1, 400):
            r = compact_rounds(a, b, G, L, r, 1, one=True)
            both(a, b, lambda e: e.missing_decisions(lane, gids, size_limit=lim, too_much_gap=lim + 1),
                 f"missing decisions lane {lane} size_limit {lim}")
    return r


def group_flags(a, b, L, r):
    """get / select / clear group flags at every lane, each call with VALID records"""
    gids = np.arange(G, dtype=np.uint32)
    for lane in range(L):
        r = compact_rounds(a, b, G, L, r, 1, one=True)
        both(a, b, lambda e: e.group_flags(gids, lane), f"group flags lane {lane}")
        for mask, value in ((abi.GF_NOT_CAUGHT_UP, 0), (abi.GF_NOT_CAUGHT_UP, abi.GF_NOT_CAUGHT_UP), (0, 0),
                            (abi.GF_NEEDS_SYNC, abi.GF_NEEDS_SYNC)):
            r = compact_rounds(a, b, G, L, r, 1, one=True)
            both(a, b, lambda e: e.select_groups(lane, mask, value), f"select lane {lane} {mask}/{value}")
        r = compact_rounds(a, b, G, L, r, 1, one=True)
        for e in (a, b):
            e.clear_group_flags(lane, gids[::3], abi.GF_NOT_CAUGHT_UP | abi.GF_NEEDS_SYNC)
    return r


def destroy_create(a, b, L, r):
    """destroy VALID groups, recreate them with another member set (a lane subset and a remote member), then with the
    identity set again; then create over live VALID groups (a reset to slot 0)"""
    D = np.arange(0, G, 5, dtype=np.uint32)
    for e in (a, b):
        e.destroy_groups(D)
    same_state(a, b, G, L)  # a destroyed group's record is no longer VALID: nothing writes it back over the free rows
    r = compact_rounds(a, b, G, L, r, 2)
    other = group_descs(len(D), members=NODES[: max(1, L - 1)] + [REMOTE], prefix="Other")
    other["gid"] = D
    for e in (a, b):
        e.create_groups(other)
    r = compact_rounds(a, b, G, L, r, 3)
    ident = group_descs(len(D), members=NODES[:L], prefix="Again")
    ident["gid"] = D
    for e in (a, b):
        e.create_groups(ident)
    r = compact_rounds(a, b, G, L, r, 3)
    assert run_round(a, b, G, L, r) == 1
    E = np.arange(3, G, 10, dtype=np.uint32)
    reset = group_descs(len(E), members=NODES[:L], prefix="Reset")
    reset["gid"] = E
    for e in (a, b):
        e.create_groups(reset)
    return compact_rounds(a, b, G, L, r + 1, 2)


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.uint8).copy()).to("cuda")


def _host(t, dtype):
    return t.cpu().numpy().view(dtype).reshape(-1)


# The device forms go through wire.propose_device_heads and the DevNode calls of the two-host device test; their
# outputs are compared whole (zero-filled buffers, gpx_dev_ctl as raw bytes), so no field of the control block is
# named here.
def propose_call(e, reqs, pay, device):
    if not device:
        acc, blob, st = e.propose(reqs, pay)
        return st, as_set(acc)
    import torch
    n = len(reqs)
    st, acc = torch.zeros(n, dtype=torch.int32, device="cuda"), torch.zeros((n, 48), dtype=torch.uint8, device="cuda")
    heads, ctl = torch.zeros(n, dtype=torch.int32, device="cuda"), DevNode(e).ctl()
    wire.propose_device_heads(e, _dev(reqs), n, _dev(np.concatenate([pay, np.zeros(16, np.uint8)])), len(pay), st,
                              acc, heads, ctl)
    torch.cuda.synchronize()
    pairs = np.zeros(n, dtype=[("accept", abi.accept_dtype), ("head", "<i4")])  # each ACCEPT with its head
    pairs["accept"], pairs["head"] = _host(acc, abi.accept_dtype), heads.cpu().numpy()
    return st.cpu().numpy(), as_set(pairs), ctl.cpu().numpy()


def accepts_call(e, acc, blob, device, fused=False):
    if fused:
        rep, dec, ex, extra = e.handle_accepts_fused(acc, blob)
        return rep, as_set(dec), ex, as_set(extra)
    if not device:
        rep, extra = e.handle_accepts(acc, blob)
        return rep, as_set(extra)
    import torch
    d = DevIn(_dev(acc), _dev(np.concatenate([blob, np.zeros(16, np.uint8)])), (len(acc), len(blob)))
    node, extra = DevNode(e), torch.zeros((4096, 24), dtype=torch.uint8, device="cuda")
    ctl = node.ctl()
    rep = node.accepts(d, ctl, extra)
    torch.cuda.synchronize()
    return rep.cpu().numpy(), as_set(_host(extra, abi.exec_dtype)), ctl.cpu().numpy()


def replies_call(e, reps, device):
    if not device:
        return as_set(e.handle_accept_replies(reps))
    import torch
    node, dec = DevNode(e), torch.zeros((len(reps), 32), dtype=torch.uint8, device="cuda")
    ctl = node.ctl()
    node.replies(_dev(reps), len(reps), dec, ctl)
    torch.cuda.synchronize()
    return as_set(_host(dec, abi.decision_dtype)), ctl.cpu().numpy()


def decisions_call(e, dec, device):
    if not device:
        ex, extra = e.handle_decisions(dec)
        return ex, as_set(extra)
    import torch
    node, extra = DevNode(e), torch.zeros((4096, 24), dtype=torch.uint8, device="cuda")
    ctl = node.ctl()
    ex = node.decisions(_dev(dec), len(dec), extra, ctl)
    torch.cuda.synchronize()
    return ex.cpu().numpy(), as_set(_host(extra, abi.exec_dtype)), ctl.cpu().numpy()


def phase_calls(a, b, L, r, device=False, fused=False):
    """each phase call on a quarter of the groups while their records are VALID (a compacting round before each):
    proposals at the coordinator's next slot; a remote coordinator's ACCEPTs at a higher ballot for the acceptors'
    next slot; ACCEPT_REPLYs carrying a higher ballot to the coordinator (preemption); DECISIONs for the next slot"""
    rng = np.random.default_rng(r)
    P, A, T, D = (np.arange(k, G, 4, dtype=np.uint32) for k in range(4))
    reqs, pay = make_requests(P, payload_len=5, seed=91, round_no=r, entry_lane=r % L, entry_node=NODES[r % L])
    r = compact_rounds(a, b, G, L, r, 1, one=True)
    both(a, b, lambda e: propose_call(e, reqs, pay, device), "proposals")

    r = compact_rounds(a, b, G, L, r, 1)
    _, row = coord_view(b, A, L)
    acc = np.zeros(len(A), dtype=abi.accept_dtype)
    acc["gid"], acc["slot"] = A, row["acc_slot"]
    acc["bnum"], acc["bcoord"] = wrap32(row["acc_bnum"].astype(np.int64) + 1), REMOTE
    acc["median_cp"] = wrap32(row["acc_slot"].astype(np.int64) - 2)
    acc["flags"], acc["dst_mask"] = abi.F_ACCEPT, (1 << L) - 1
    acc["req_id"] = rng.integers(1, 1 << 60, size=len(A))
    acc["payload_off"] = np.arange(len(A)) * 16
    acc["payload_len"], acc["nreq"], acc["sender"] = 7, 1, REMOTE
    blob = rng.integers(48, 122, size=16 * len(A)).astype(np.uint8)
    both(a, b, lambda e: accepts_call(e, acc, blob, device, fused), "accept replies")

    r = compact_rounds(a, b, G, L, r, 1)
    cl, row = coord_view(b, T, L)
    rep = np.zeros(len(T), dtype=abi.reply_dtype)
    rep["gid"], rep["slot"] = T, wrap32(row["acc_slot"].astype(np.int64) - 1)
    rep["bnum"], rep["bcoord"] = wrap32(row["acc_bnum"].astype(np.int64) + 1), REMOTE
    rep["max_cp"] = wrap32(row["acc_slot"].astype(np.int64) - 2)
    rep["who"] = [abi.who(int(m), int(c), abi.F_NACK) for m, c in zip((cl + 1) % L, cl)]
    rep["req_id"] = rng.integers(1, 1 << 60, size=len(T))
    both(a, b, lambda e: replies_call(e, rep, device), "decisions from replies")

    r = compact_rounds(a, b, G, L, r, 1)
    _, row = coord_view(b, D, L)
    dec = np.zeros(len(D), dtype=abi.decision_dtype)
    dec["gid"], dec["slot"] = D, row["acc_slot"]
    dec["bnum"], dec["bcoord"] = row["acc_bnum"], row["acc_bcoord"]
    dec["median_cp"] = wrap32(row["acc_slot"].astype(np.int64) - 2)
    dec["flags"], dec["dst_mask"] = abi.F_DECISION, (1 << L) - 1
    dec["req_id"] = rng.integers(1, 1 << 60, size=len(D))
    both(a, b, lambda e: decisions_call(e, dec, device), "decision EXEC rows")
    return compact_rounds(a, b, G, L, r, 3)


def compact_device_round(a, b, L, r):
    """gpx_round_device_compact (k_propose + k_act, or the four phase kernels) with VALID records"""
    import torch
    reqs, pay = plain_requests(G, L, r)

    def go(e):
        n = len(reqs)
        d_reqs, d_pay = _dev(reqs), _dev(np.concatenate([pay, np.zeros(16, np.uint8)]))
        st = torch.zeros(n, dtype=torch.int32, device="cuda")
        ex = torch.zeros(n * L * abi.exec_dtype.itemsize, dtype=torch.uint8, device="cuda")
        bufs = abi.DevRoundBufs(d_reqs.data_ptr(), d_pay.data_ptr(), len(pay), n, st.data_ptr(), ex.data_ptr())
        e.L.check(e.L.fn("round_device_compact")(e.handle, C.byref(bufs), None))
        torch.cuda.synchronize()
        x = ex.cpu().numpy().view(abi.exec_dtype).copy()
        x["payload_off"] = 0
        return st.cpu().numpy(), as_set(x)
    both(a, b, go, "compact device round")
    return compact_rounds(a, b, G, L, r + 1, 2)


def pipeline(a, b, L, r):
    """gpx_round_submit with packed requests and compact summaries, up to GPX_PIPE_DEPTH rounds in flight, then a
    dump; then one pipelined round on the team kernel of the compacting engine (launch_round settles for it)"""
    tickets = []
    for k in range(abi.PIPE_DEPTH):
        reqs, pay = plain_requests(G, L, r + k)
        pk = np.zeros(len(reqs), dtype=abi.request_packed_dtype)
        pk["gid"], pk["payload_len"], pk["req_id"] = reqs["gid"], reqs["payload_len"], reqs["req_id"]
        pk["flags"] = reqs["flags"]
        packed = np.concatenate([pay[o: o + 1] for o in reqs["payload_off"]])
        tickets.append([(e, e.round_submit(pk, packed, compact=True, packed=True)) for e in (a, b)])
    for ts in tickets:
        (ea, ta), (eb, tb) = ts
        sa, sb = ea.round_wait(ta), eb.round_wait(tb)
        assert sa["sum"].tobytes() == sb["sum"].tobytes(), "compact summaries"
        assert as_set(sa["extra"]) == as_set(sb["extra"]), "extra queue"
    r += abi.PIPE_DEPTH
    same_state(a, b, G, L)
    r = compact_rounds(a, b, G, L, r, 2, one=True)
    set_mode(a, TEAM)
    reqs, pay = plain_requests(G, L, r)
    ta, tb = a.round_submit(reqs, pay), b.round_submit(reqs, pay)
    sa, sb = a.round_wait(ta), b.round_wait(tb)
    assert sa["status"].tobytes() == sb["status"].tobytes() and sa["exec"].tobytes() == sb["exec"].tobytes()
    set_mode(a, 0)
    return compact_rounds(a, b, G, L, r + 1, 2)


def host_slow_kernel(a, b, L, r, eo=None):
    """round mode 2 (host-launched k_round_slow after k_round_g): a second request for some groups and STOPs for others,
    so that groups whose record is VALID leave the fast path; the rounds equal the oracle's"""
    set_mode(a, THREAD_HOST)
    for _ in range(2):
        r = trio_round(a, b, eo, L, r)
    gids = np.repeat(np.arange(G), np.where(np.arange(G) % 4 == 1, 2, 1))
    stop = np.zeros(len(gids), dtype=bool)
    stop[np.nonzero(gids % 9 == 4)[0]] = True
    r = trio_round(a, b, eo, L, r, make_requests(gids, payload_len=3, seed=5, round_no=r, stop_mask=stop,
                                                 entry_lane=r % L, entry_node=NODES[r % L]))
    for _ in range(2):
        r = trio_round(a, b, eo, L, r)
    same_as_oracle(a, eo, L)
    assert a.counters()["stops_executed"] > 0
    set_mode(a, 0)
    return r


def kernel_timing(a, b, L, r):
    """kernel timing on across compacting rounds (the settle runs outside the timed window), then a state call"""
    for e in (a, b):
        e.L.check(e.L.fn("enable_kernel_timing")(e.handle, C.c_int(1)))
    r = compact_rounds(a, b, G, L, r, 3, one=True)
    same_state(a, b, G, L)
    r = compact_rounds(a, b, G, L, r, 2, one=True)
    r = compact_device_round(a, b, L, r)
    for e in (a, b):
        e.L.check(e.L.fn("enable_kernel_timing")(e.handle, C.c_int(0)))
    return r


CALLS = {
    "view_change": view_change,
    "missing_decisions": missing_decisions,
    "group_flags": group_flags,
    "destroy_create": destroy_create,
    "phase_calls": phase_calls,
    "device_phase_calls": lambda a, b, L, r: phase_calls(a, b, L, r, device=True),
    "accepts_fused": lambda a, b, L, r: phase_calls(a, b, L, r, fused=True),
    "compact_device_round": compact_device_round,
    "pipeline": pipeline,
    "host_slow_kernel": host_slow_kernel,
    "kernel_timing": kernel_timing,
}
ORACLE_CALLS = ("view_change", "host_slow_kernel")  # also run on a CPU oracle engine
LAYOUTS = [(1, None), (2, None), (3, None), (1, "intmax"), (2, "intmax"), (3, "intmax")]


@pytest.mark.parametrize("L,base", LAYOUTS)
@pytest.mark.parametrize("call", list(CALLS))
def test_call_while_records_are_valid(cuda_lib, oracle_lib, call, L, base):
    a, b = twins(cuda_lib, L, G, None if base is None else SLOT_BASES[base])
    if call in ORACLE_CALLS:
        eo = oracle_twin(oracle_lib, a, L, base)
        r = 0
        for _ in range(2):
            k0 = a.counters()["kernel_launches"]
            r = trio_round(a, b, eo, L, r)
            assert a.counters()["kernel_launches"] - k0 == 1
        r = CALLS[call](a, b, L, r, eo)
        eo.close()
    else:
        r = compact_rounds(a, b, G, L, 0, 2, one=True)
        r = CALLS[call](a, b, L, r)
    r = compact_rounds(a, b, G, L, r, 2)
    same_state(a, b, G, L)
    compare_logs(a, b, L)
    if call in ("missing_decisions", "group_flags", "destroy_create"):
        same_rings(a, b, L)  # only in-order rounds logged: byte for byte
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("L,base", LAYOUTS)
def test_forwards_encoders_while_records_are_valid(cuda_lib, L, base):
    """the forwards encoders settle nothing: after a round in which identity groups compact and the groups whose
    coordinator is a remote member forward their requests, gpx_wire_encode_forwards_device and
    gpx_wire_encode_json_sweep_device on that round's statuses -- before any call that settles -- give the same rstatus
    and bytes on both twins (propose_route reads only ballots and EXISTS, which a VALID record keeps current)"""
    import torch
    a, b = engines(cuda_lib, L, G, None if base is None else SLOT_BASES[base])
    n_rem = G // 5
    gids = np.arange(G, dtype=np.uint32)
    names = group_names(G - n_rem) + group_names(n_rem, "RemoteApp")
    for e in (a, b):
        wire.set_group_names(e, gids, names)
    sent = 0
    for r in range(6):
        reqs, pay = plain_requests(G, L, r)
        meta = np.zeros(len(reqs), abi.req_meta_dtype)
        meta["client_ip"], meta["client_port"], meta["entry_time"] = [10, 1, 2, 3], 4567, 1000 + r
        d_reqs, d_meta, d_pay = _dev(reqs), _dev(meta), _dev(np.concatenate([pay, np.zeros(16, np.uint8)]))
        outs = []
        for e in (a, b):
            n = len(reqs)
            st = torch.zeros(n, dtype=torch.int32, device="cuda")
            ex = torch.zeros(n * L * abi.exec_dtype.itemsize, dtype=torch.uint8, device="cuda")
            bufs = abi.DevRoundBufs(d_reqs.data_ptr(), d_pay.data_ptr(), len(pay), n, st.data_ptr(), ex.data_ptr())
            e.L.check(e.L.fn("round_device")(e.handle, C.byref(bufs), None))
            fw = wire.encode_forwards_device(e, d_reqs, d_meta, n, st, d_pay, [], (1, 1))
            sw = wire.encode_json_sweep_device(e, None, 0, None, None, 0, d_reqs, d_meta, n, st, d_pay, [], (1, 1))
            torch.cuda.synchronize()
            outs.append([t.cpu().numpy().tobytes() for t in (st, ex, fw.rstatus, fw.out, fw.refs, sw.rstatus_reqs,
                                                             sw.out, sw.refs)])
        for i, what in enumerate(("status", "EXEC rows", "forwards rstatus", "forward packets", "forward refs",
                                  "sweep rstatus", "sweep packets", "sweep refs")):
            assert outs[0][i] == outs[1][i], f"round {r}: {what}"
        rs = np.frombuffer(outs[0][2], np.uint8)
        sent += int((rs == abi.WE_SENT).sum())
    assert sent > 0, "some requests were forwarded to a remote coordinator"
    same_state(a, b, G, L)
    compare_logs(a, b, L)
    for e in (a, b):
        e.close()


MIXED = [None, [100, 101], [102, 100, 101], [101, 102, 900], [100]]


def mixed_members(L):
    """the five member sets, identity = the L lanes"""
    return [NODES[:L] if m is None else m for m in MIXED]


@pytest.mark.parametrize("seed", [3, 4])
def test_mixed_layouts_against_the_oracle(oracle_lib, cuda_lib, seed):
    """identity groups (which compact in the long stretches of in-order rounds) beside lane subsets, permuted and remote
    members, in the adversarial schedule with PREPAREs: every output of every call equals the oracle's"""
    f = Fuzzer([oracle_lib, cuda_lib], G=600, R=3, W=8, seed=seed, lane_node=NODES[:3], members=mixed_members(3))
    # stretches of in-order rounds (one request per group: the identity groups compact), each followed by a call
    # that settles -- PREPAREs, the phase steps, dump / flags -- and then the adversarial schedule
    for k in range(8):
        for _ in range(3):
            f.step_round(frac=1.0, max_per_group=1)
        (f.step_prepares, f.step_accepts, f.step_replies, f.step_decisions, f.check_state)[k % 5]()
    f.check_state()
    f.run(steps=50, rival=True, view_changes=True, round_prob=0.8, prepares=True, check_every=5)
    f.close()


@pytest.mark.parametrize("L", [2, 3])
def test_mixed_layouts_against_the_team_kernel(cuda_lib, L):
    """the same layouts on twin engines (k_round_g and the team kernel), plain in-order rounds with a state call every
    few rounds: rows byte for byte, and the rows of non-identity groups and of non-member lanes are never touched by
    a settle (they only change in a round that gives their group a request)"""
    Gm = 3000
    lane_node = NODES[:L]
    sets = [m for m in mixed_members(L) if any(x in lane_node for x in m)]
    cfg = dict(max_groups=Gm, n_lanes=L, lane_node=lane_node, window=8, max_group_size=3, max_batch_recs=1 << 14,
               max_batch_payload=1 << 21, log_ring_bytes=1 << 24, checkpoint_interval=4)
    es = [Engine(cuda_lib, make_config(cuda_lib, **cfg)) for _ in range(2)]
    set_mode(es[1], TEAM)
    d = group_descs(Gm, members=())
    for g in range(Gm):
        m = sets[g % len(sets)]
        d["n_members"][g], d["members"][g, : len(m)] = len(m), m
    for e in es:
        e.create_groups(d)
    a, b = es
    ident = np.array([sorted(sets[g % len(sets)]) == sorted(lane_node) for g in range(Gm)])
    gids = np.arange(Gm, dtype=np.uint32)
    calls = [lambda e: e.group_flags(gids, 0), lambda e: e.select_groups(L - 1, abi.GF_NOT_CAUGHT_UP, 0),
             lambda e: e.missing_decisions(0, gids, size_limit=1, too_much_gap=2),
             lambda e: e.pause_groups(gids[1::97])[1]]
    for r in range(24):
        # identity groups every round; the others only on even rounds, so odd rounds leave their rows alone
        sel = gids if r % 2 == 0 else gids[ident]
        reqs, pay = make_requests(sel, payload_len=2, seed=33, round_no=r, entry_lane=r % L, entry_node=NODES[r % L])
        before = [b.dump_rows(gids[~ident], l) for l in range(L)] if r % 2 else None
        run_round(a, b, Gm, L, r, (reqs, pay))
        if before is not None:
            for l in range(L):
                got = a.dump_rows(gids[~ident], l)
                assert got.tobytes() == before[l].tobytes(), f"round {r}: rows of non-identity groups, lane {l}"
        if r % 3 == 2:
            both(a, b, calls[(r // 3) % len(calls)], f"state call after round {r}")
    same_state(a, b, Gm, L)
    compare_logs(a, b, L)
    for e in es:
        e.close()
