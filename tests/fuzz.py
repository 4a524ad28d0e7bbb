"""Adversarial schedule generator for the per-phase API.

Drives one or two engines in lock step through a lossy, duplicating, reordering "network":
records produced by one phase sit in pools and are delivered later in random batches
(grouped by gid, random order inside a group).  It injects the cases SURVEY.md 8a lists:
higher-ballot accepts from a rival coordinator (NACKs, preemption), duplicate accepts and
replies, out-of-order and duplicate decisions, commits that overtake their accepts
(placeholder + reconstructDecision), accepts at or below the GC slot, STOP requests,
coordinator change patches, multi-record runs per group in one batch.

slot_base / ballot_base move every group's slots and ballot numbers by a fixed offset modulo 2^32 before the first
step (tests/wrap_cases.py), so that a run crosses the Java int wrap.  The bookkeeping (max_proposed, rival_bnum,
history, the slots of view changes) stays unwrapped, as at offset 0; slots and ballots are wrapped where records and
patches are built and unwrapped where rows and EXEC records are read.  At offset 0 every draw and record is the same
as without the offsets.

lane_node / members give the engine's layout (tests/layout_cases.py): the node each lane serves, in any order, and the
member lists of the groups (gid g gets members[g % len(members)]), which may name nodes no lane serves.  Everything
that depends on the layout follows from it: the initial coordinator (roundRobinCoordinator over the sorted members,
at a lane or remote), the lanes a record is addressed to (the group's member lanes), the rival coordinators and
PREPARE senders (members), view changes (patches at the member lanes, the new coordinator a local member), lost
destinations (member lanes).  Each remote member is a minimal acceptor: it acks every ACCEPT a local coordinator sent
whose ballot is not below its promise, with its own member index, so a group whose local members are a minority
still decides.  Without a layout, lane l serves NODES[l] and every group's members are the R lanes.

With two engines every output of every call is compared bit-exactly (streams whose
inter-group order is scheduling-dependent on the device are compared after a stable sort by
gid; the per-group order is protocol-defined and must match).
"""
from __future__ import annotations

import numpy as np

from helpers import Engine, abi, canon, group_descs, make_config, make_requests
from wrap_cases import shift_rows, unwrap, wrap32

NODES = [100, 101, 102, 103, 104]


def _eq(a: np.ndarray, b: np.ndarray, what: str, skip=()):
    assert len(a) == len(b), f"{what}: length {len(a)} != {len(b)}"
    for f in a.dtype.names:
        if f in skip:
            continue
        x, y = a[f], b[f]
        if f == "payload_off" and a.dtype == abi.exec_dtype:
            # the log position of a BATCHED slot's blob depends on the order in which the device's blocks reserved
            # space for constructed blobs inside one fused round (content and length are compared through the log)
            single = (a["flags"] >> 16) <= 1
            x, y = x[single], y[single]
        if not np.array_equal(x, y):
            bad = np.nonzero(a[f] != b[f])[0][:5]
            raise AssertionError(f"{what}: field {f} differs at {bad}: {a[bad]} vs {b[bad]}")


class Fuzzer:
    def __init__(self, libs, G=64, R=3, W=8, seed=1, slot_base=0, ballot_base=0, lane_node=None, members=None, **cfg):
        self.rng = np.random.default_rng(seed)
        self.G, self.R, self.W = G, R, W
        self.slot_base, self.ballot_base = int(slot_base), int(ballot_base)
        self.lane_node = list(NODES[:R] if lane_node is None else lane_node)
        self.L = len(self.lane_node)
        sets = [tuple(NODES[:R])] if members is None else [tuple(m) for m in members]
        lane_of = {n: l for l, n in enumerate(self.lane_node)}
        self.members = [sorted(sets[g % len(sets)]) for g in range(G)]  # PISM ctor sorts groupMembers
        self.mlanes = [[lane_of[m] for m in mem if m in lane_of] for mem in self.members]  # member lanes, member order
        assert all(self.mlanes), "every group needs a member at some lane"
        self.lane_mask = np.array([sum(1 << l for l in ml) for ml in self.mlanes])
        kw = dict(max_groups=G, n_lanes=self.L, lane_node=self.lane_node, window=W,
                  max_group_size=max(len(m) for m in sets), max_batch_recs=1 << 14, max_batch_payload=1 << 20,
                  log_ring_bytes=1 << 27)
        kw.update(cfg)
        self.engines = [Engine(l, make_config(l, **kw)) for l in libs]
        d = group_descs(G, members=())
        for g in range(G):  # as listed, unsorted
            m = sets[g % len(sets)]
            d["n_members"][g] = len(m)
            d["members"][g, :len(m)] = m
        for e in self.engines:
            e.create_groups(d)
        if self.slot_base or self.ballot_base:
            gids = np.arange(G)
            rows = np.concatenate([self.engines[0].dump_rows(gids, l) for l in range(self.L)])
            rows = rows[(self.lane_mask[rows["gid"]] >> rows["lane"].astype(np.int64)) & 1 == 1]
            rows = shift_rows(rows, self.slot_base, self.ballot_base)
            for e in self.engines:
                e.load_rows(rows)
        self.coord_idx = np.array([abs(abi.java_string_hash(f"NoopPaxosApp{g}")) % len(self.members[g])
                                   for g in range(G)])  # member index
        # remote members: member index -> promised (unwrapped ballot number, coordinator); createHRI's (0, coordinator)
        self.promise = [{i: (0, mem[self.coord_idx[g]]) for i, m in enumerate(mem) if m not in lane_of}
                        for g, mem in enumerate(self.members)]
        self.n_forward = 0  # requests answered GPX_RS_FORWARD (the coordinator is remote)
        self.acc_pool = []   # (rec, blob bytes)
        self.rep_pool = []
        self.dec_pool = []
        self.round_no = 0
        self.history = [dict() for _ in range(self.L)]  # lane -> gid -> [(slot, req_id)]
        self.stopped = set()
        self.rival_bnum = np.zeros(G, dtype=np.int64)
        self.max_proposed = np.zeros(G, dtype=np.int64)  # highest slot any coordinator issued an ACCEPT for

    # ---- wire values <-> unwrapped bookkeeping -------------------------------------------
    def ws(self, s):
        return wrap32(s + self.slot_base)

    def us(self, s):
        return unwrap(s, self.slot_base)

    def wb(self, b):
        return wrap32(b + self.ballot_base)

    def ub(self, b):
        return unwrap(b, self.ballot_base)

    # ---- comparison helpers ----------------------------------------------------------
    def _all(self, fn):
        outs = [fn(e) for e in self.engines]
        return outs

    def member_lane(self, g):
        """one of the group's member lanes, drawn at random (a lost destination)"""
        ml = self.mlanes[g]
        return ml[int(self.rng.integers(0, len(ml)))]

    def member_rows(self):
        """every group's row at its first member lane (lane 0 for all groups without a layout)"""
        gids = np.arange(self.G)
        first = np.array([min(ml) for ml in self.mlanes])
        rows = None
        for l in np.unique(first):
            r = self.engines[0].dump_rows(gids, int(l))
            if rows is None:
                rows = r
            rows[first == l] = r[first == l]
        return rows

    def check_state(self):
        if len(self.engines) < 2:
            return
        gids = np.arange(self.G)
        for l in range(self.L):
            rows = [e.dump_rows(gids, l) for e in self.engines]
            _eq(rows[0], rows[1], f"rows lane {l}")
            fl = [e.group_flags(gids, l) for e in self.engines]
            assert np.array_equal(fl[0], fl[1]), f"group flags lane {l}"
            heads = [e.log_head(l) for e in self.engines]
            assert heads[0] == heads[1], f"log ring heads lane {l}: {heads}"
        c = [e.counters() for e in self.engines]
        for x in c:
            x.pop("kernel_launches")
        assert c[0] == c[1], f"counters differ: { {k: (c[0][k], c[1][k]) for k in c[0] if c[0][k] != c[1][k]} }"

    def record_exec(self, ex):
        # EXEC records of one call are applied per group in slot order: the primary record of a
        # decision and the extra records released by the same call interleave (include/gpx.h)
        ex = ex[(ex["flags"] & abi.F_VOID) == 0]
        ex = ex[np.lexsort((self.us(ex["slot"]), ex["gid"]))]
        for x in ex:
            lane = int((x["flags"] >> 12) & 0xF)
            assert (int(self.lane_mask[int(x["gid"])]) >> lane) & 1, f"lane {lane} executed gid {x['gid']}, not a member"
            h = self.history[lane].setdefault(int(x["gid"]), [])
            h.append((self.us(int(x["slot"])), int(x["req_id"])))
            if x["flags"] & abi.F_STOP:
                self.stopped.add(int(x["gid"]))

    # ---- phases ------------------------------------------------------------------------
    def step_propose(self, frac=0.5, stop_prob=0.0, max_per_group=3):
        rng = self.rng
        gsel = np.nonzero(rng.random(self.G) < frac)[0]
        if len(gsel) == 0:
            return
        cnt = rng.integers(1, max_per_group + 1, size=len(gsel))
        gids = np.repeat(gsel, cnt)
        lens = rng.integers(1, 48, size=len(gids))
        stop = rng.random(len(gids)) < stop_prob
        entry = int(rng.integers(0, self.L))
        reqs, pay = make_requests(gids, payload_len=lens, seed=77, round_no=self.round_no, entry_lane=entry,
                                  entry_node=self.lane_node[entry], stop_mask=stop)
        self.round_no += 1
        outs = self._all(lambda e: e.propose(reqs, pay))
        acc0, blob0, st0 = outs[0]
        self.n_forward += int((st0 == abi.RS_FORWARD).sum())
        for acc, blob, st in outs[1:]:
            assert np.array_equal(st0, st), f"propose status: {st0} vs {st}"
            a, b = canon(acc0), canon(acc)
            _eq(a, b, "accepts", skip=("payload_off",))
            for x, y in zip(a, b):
                ox, oy, ln = int(x["payload_off"]), int(y["payload_off"]), int(x["payload_len"])
                assert np.array_equal(blob0[ox: ox + ln], blob[oy: oy + ln]), "accept blob bytes"
                if x["nreq"] == 1:
                    assert ox == oy
        for x in canon(acc0):
            o, ln = int(x["payload_off"]), int(x["payload_len"])
            self.acc_pool.append((x.copy(), blob0[o: o + ln].copy()))
            self.max_proposed[int(x["gid"])] = max(self.max_proposed[int(x["gid"])], self.us(int(x["slot"])))

    def step_round(self, frac=0.5, stop_prob=0.0, max_per_group=3, fn="round"):
        """one fused round (gpx_round / k_round) in whatever state the adversarial phase steps left the groups:
        outstanding proposals, NACKed ballots, resigned or pre-active coordinators, placeholders, stopped groups"""
        rng = self.rng
        gsel = np.nonzero(rng.random(self.G) < frac)[0]
        if len(gsel) == 0:
            return
        cnt = rng.integers(1, max_per_group + 1, size=len(gsel))
        gids = np.repeat(gsel, cnt)
        lens = rng.integers(1, 48, size=len(gids))
        stop = rng.random(len(gids)) < stop_prob
        entry = int(rng.integers(0, self.L))
        reqs, pay = make_requests(gids, payload_len=lens, seed=79, round_no=self.round_no, entry_lane=entry,
                                  entry_node=self.lane_node[entry], stop_mask=stop)
        self.round_no += 1
        cap = 4 * len(reqs) * self.L + 256
        outs = self._all(lambda e: getattr(e, fn)(reqs, pay, extra_cap=cap))
        st0, ex0, xt0 = outs[0]
        self.n_forward += int((st0 == abi.RS_FORWARD).sum())
        key = lambda r: r[np.lexsort((r["slot"], r["gid"], (r["flags"] >> 12) & 0xF))]
        live = lambda r: r[(r["flags"] & abi.F_VOID) == 0]
        a0 = key(live(np.concatenate([ex0, xt0])))
        for st, ex, xt in outs[1:]:
            assert np.array_equal(st0, st), f"round status: {st0} vs {st}"
            a = key(live(np.concatenate([ex, xt])))
            assert len(a0) == len(a), f"round executions {len(a0)} vs {len(a)}"
            for f in ("gid", "slot", "req_id"):
                assert np.array_equal(a0[f], a[f]), f"round exec {f}"
            assert np.array_equal(a0["flags"] & ~np.uint32(abi.F_EXTRA), a["flags"] & ~np.uint32(abi.F_EXTRA)), "round exec flags"
        # a status is a slot or a GPX_RS_* code, and a wrapped slot may equal a code.  Unwrapped, every slot is > 0; a
        # code may unwrap to a small positive number too and then counts as a slot: max_proposed only has to bound
        # the slots issued from above (view changes start beyond it)
        ust = self.us(st0)
        ok = ust > 0
        for g, sl in zip(reqs["gid"][ok], ust[ok]):
            self.max_proposed[int(g)] = max(self.max_proposed[int(g)], int(sl))
        self.record_exec(np.concatenate([ex0, xt0]))

    def inject_rival_accepts(self, n=4):
        """A rival coordinator (another member, higher ballot number) re-proposes slots."""
        rng = self.rng
        rows = self.member_rows()
        for _ in range(n):
            g = int(rng.integers(0, self.G))
            if g in self.stopped:
                continue
            self.rival_bnum[g] += 1
            mem = self.members[g]
            rival = mem[(self.coord_idx[g] + 1) % len(mem)]
            acc_slot = self.us(int(rows[g]["acc_slot"]))
            slot = acc_slot + int(rng.integers(-2, 3))
            rec = np.zeros(1, dtype=abi.accept_dtype)[0]
            rec["gid"], rec["slot"], rec["bnum"], rec["bcoord"] = g, self.ws(slot), self.wb(int(self.rival_bnum[g])), rival
            rec["median_cp"] = self.ws(acc_slot - int(rng.integers(1, 4)))
            rec["flags"] = abi.F_ACCEPT
            rec["dst_mask"] = self.lane_mask[g]
            rec["req_id"] = int(rng.integers(1, 1 << 60))
            ln = int(rng.integers(1, 33))
            rec["payload_len"], rec["nreq"], rec["sender"] = ln, 1, rival
            blob = rng.integers(48, 122, size=ln).astype(np.uint8)
            self.acc_pool.append((rec, blob))

    def step_prepares(self, n=3):
        """phase 1a: would-be coordinators (any member) send PREPAREs with a fresh ballot -- or a stale one -- and a
        firstUndecidedSlot around the acceptors' slots, to a subset of the lanes; the replies (ballot, firstSlot,
        accepted pvalues in slot order, NACK / LOGGED / FROM_LOG flags) and the logged PREPARE images must agree"""
        rng = self.rng
        rows = self.member_rows()
        recs = []
        for _ in range(n):
            g = int(rng.integers(0, self.G))
            node = self.members[g][int(rng.integers(0, len(self.members[g])))]
            if rng.random() < 0.7:
                self.rival_bnum[g] += 1
                bn = int(self.rival_bnum[g])
            else:
                bn = int(self.rival_bnum[g]) - int(rng.integers(0, 3))  # stale or equal ballot: NACK / plain ack
            r = np.zeros(1, dtype=abi.decision_dtype)[0]
            r["gid"], r["bnum"], r["bcoord"] = g, self.wb(bn), node
            r["slot"] = self.ws(self.us(int(rows[g]["acc_slot"])) + int(rng.integers(-3, 3)))
            r["flags"] = abi.F_PREPARE
            mask = int(self.lane_mask[g])
            if rng.random() < 0.3:
                mask &= ~(1 << self.member_lane(g))  # the multicast loses a destination
            r["dst_mask"] = mask
            recs.append(r)
            self.promise_remote(g, (bn, node))
        recs.sort(key=lambda r: int(r["gid"]))
        recs = np.array(recs, dtype=abi.decision_dtype)
        outs = self._all(lambda e: e.handle_prepares(recs))
        r0 = outs[0]
        for r1 in outs[1:]:
            for f in ("gid", "first_slot", "bnum", "bcoord", "who", "n_accepted"):
                assert np.array_equal(r0[f], r1[f]), f"prepare reply {f}: {r0[f]} vs {r1[f]}"
            for a, b in zip(r0, r1):
                k = int(a["n_accepted"])
                for f in abi.accepted_pvalue_dtype.names:
                    x, y = a["accepted"][f][:k], b["accepted"][f][:k]
                    if f == "frame_ref":  # batched blobs: position depends on block scheduling inside a fused round
                        single = (a["accepted"]["flags"][:k] >> 16) <= 1
                        x, y = x[single], y[single]
                    assert np.array_equal(x, y), f"prepare reply accepted.{f}"
                assert not b["accepted"][k:].view(np.uint8).any(), "entries beyond n_accepted must be zero"

    def _take(self, pool, p_deliver, p_dup, p_keep):
        rng = self.rng
        batch, rest = [], []
        for item in pool:
            u = rng.random()
            if u < p_deliver:
                batch.append(item)
                if rng.random() < p_dup:
                    batch.append(item)
                if rng.random() < p_keep:
                    rest.append(item)  # will be delivered again later (late duplicate)
            else:
                rest.append(item)
        pool[:] = rest
        rng.shuffle(batch)
        return batch

    def step_accepts(self, p_deliver=0.7, p_dup=0.1, p_keep=0.05, lane_loss=0.1):
        batch = self._take(self.acc_pool, p_deliver, p_dup, p_keep)
        if not batch:
            return
        batch.sort(key=lambda it: int(it[0]["gid"]))  # grouped by gid, random order inside (stable sort)
        recs = np.zeros(len(batch), dtype=abi.accept_dtype)
        chunks, off = [], 0
        for i, (r, blob) in enumerate(batch):
            recs[i] = r
            recs[i]["payload_off"] = off
            pad = (-len(blob)) % 16
            chunks.append(blob)
            chunks.append(np.zeros(pad, dtype=np.uint8))
            off += len(blob) + pad
            if self.rng.random() < lane_loss:  # the multicast lost one destination
                recs[i]["dst_mask"] = int(recs[i]["dst_mask"]) & ~(1 << self.member_lane(int(recs[i]["gid"])))
        arena = np.concatenate(chunks) if chunks else np.zeros(0, np.uint8)
        outs = self._all(lambda e: e.handle_accepts(recs, arena))
        rep0, ext0 = outs[0]
        for rep, ext in outs[1:]:
            _eq(rep0, rep, "accept replies")
            _eq(canon(ext0), canon(ext), "accept-path extra exec", skip=("payload_off",))
        self.record_exec(ext0)
        for r in canon(rep0):
            self.rep_pool.append(r.copy())
        self.remote_acks(recs)

    def step_accepts_fused(self, p_deliver=0.7, p_dup=0.1, p_keep=0.05, lane_loss=0.1):
        """The loopback path: accept -> tally -> commit per ACCEPT (gpx_handle_accepts_fused / k_act)."""
        batch = self._take(self.acc_pool, p_deliver, p_dup, p_keep)
        if not batch:
            return
        batch.sort(key=lambda it: int(it[0]["gid"]))
        recs = np.zeros(len(batch), dtype=abi.accept_dtype)
        chunks, off = [], 0
        for i, (r, blob) in enumerate(batch):
            recs[i] = r
            recs[i]["payload_off"] = off
            pad = (-len(blob)) % 16
            chunks.append(blob)
            chunks.append(np.zeros(pad, dtype=np.uint8))
            off += len(blob) + pad
            if self.rng.random() < lane_loss:
                recs[i]["dst_mask"] = int(recs[i]["dst_mask"]) & ~(1 << self.member_lane(int(recs[i]["gid"])))
        arena = np.concatenate(chunks) if chunks else np.zeros(0, np.uint8)
        outs = self._all(lambda e: e.handle_accepts_fused(recs, arena))
        rep0, dec0, ex0, ext0 = outs[0]
        for rep, dec, ex, ext in outs[1:]:
            _eq(rep0, rep, "fused: leftover replies")
            _eq(dec0, dec, "fused: decisions")
            _eq(ex0, ex, "fused: exec")
            _eq(canon(ext0), canon(ext), "fused: extra exec", skip=("payload_off",))
        self.record_exec(np.concatenate([ex0, ext0]))
        for r in canon(rep0):
            self.rep_pool.append(r.copy())
        self.remote_acks(recs)

    def promise_remote(self, g, ballot):
        for i, b in self.promise[g].items():
            self.promise[g][i] = max(b, ballot)

    def remote_acks(self, recs):
        """the remote members' replies to the delivered ACCEPTs a local coordinator sent: an ack where the ballot is
        not below the member's promise, which it then adopts; maxCheckpointedSlot as executed by the slowest local
        member"""
        local = set(self.lane_node)
        for r in recs:
            g = int(r["gid"])
            if not self.promise[g] or int(r["sender"]) not in local:
                continue
            b = (self.ub(int(r["bnum"])), int(r["bcoord"]))
            dst = self.members[g].index(int(r["sender"]))
            done = [self.history[l].get(g, [(0, 0)])[-1][0] for l in self.mlanes[g]]
            for i, p in self.promise[g].items():
                if b < p:
                    continue
                self.promise[g][i] = b
                rep = np.zeros(1, dtype=abi.reply_dtype)[0]
                rep["gid"], rep["slot"], rep["bnum"], rep["bcoord"] = g, r["slot"], r["bnum"], r["bcoord"]
                rep["max_cp"] = self.ws(min(done))
                rep["who"] = i | (dst << 8)
                rep["req_id"] = r["req_id"]
                self.rep_pool.append(rep)

    def step_replies(self, p_deliver=0.7, p_dup=0.15, p_keep=0.05):
        batch = self._take(self.rep_pool, p_deliver, p_dup, p_keep)
        if not batch:
            return
        batch.sort(key=lambda r: int(r["gid"]))
        recs = np.array(batch, dtype=abi.reply_dtype)
        outs = self._all(lambda e: e.handle_accept_replies(recs))
        for d in outs[1:]:
            _eq(canon(outs[0]), canon(d), "decisions")
        for d in canon(outs[0]):
            self.dec_pool.append(d.copy())

    def step_decisions(self, p_deliver=0.7, p_dup=0.15, p_keep=0.05, lane_loss=0.1):
        batch = self._take(self.dec_pool, p_deliver, p_dup, p_keep)
        if not batch:
            return
        batch.sort(key=lambda r: int(r["gid"]))
        recs = np.array(batch, dtype=abi.decision_dtype)
        for i in range(len(recs)):
            if self.rng.random() < lane_loss:
                recs[i]["dst_mask"] = int(recs[i]["dst_mask"]) & ~(1 << self.member_lane(int(recs[i]["gid"])))
        outs = self._all(lambda e: e.handle_decisions(recs))
        ex0, ext0 = outs[0]
        for ex, ext in outs[1:]:
            _eq(ex0, ex, "exec")
            _eq(canon(ext0), canon(ext), "commit-path extra exec")
        self.record_exec(np.concatenate([ex0, ext0]))

    def patch_view_change(self, n=2):
        """Host slow path completed a coordinator change: bump acceptor ballots, resign the old
        coordinator and install an active one at another lane (effects of handlePrepare /
        handlePrepareReply as state patches, SURVEY.md 8b)."""
        rng = self.rng
        rows = [self.engines[0].dump_rows(np.arange(self.G), l) for l in range(self.L)]
        pts = []
        for _ in range(n):
            g = int(rng.integers(0, self.G))
            if g in self.stopped:
                continue
            ml = self.mlanes[g]
            cur_b = max(self.ub(int(rows[l][g]["acc_bnum"])) for l in ml)
            cur_b = max(cur_b, int(self.rival_bnum[g]))
            nb = cur_b + 1
            self.rival_bnum[g] = nb
            new_lane = self.member_lane(g)
            new_node = self.lane_node[new_lane]
            # a real view change carries over accepted pvalues (phase 1, host slow path); the fuzzer
            # stays protocol-respecting by starting the new coordinator beyond every slot any earlier
            # coordinator issued an ACCEPT for (a resigned coordinator's row no longer remembers it)
            next_slot = max(self.us(int(rows[l][g]["acc_slot"])) for l in ml)
            next_slot = max(next_slot, int(self.max_proposed[g]) + 1)
            for l in ml:
                if rows[l][g]["coord_exists"]:
                    next_slot = max(next_slot, self.us(int(rows[l][g]["next_proposal_slot"])))
            next_slot += int(rng.integers(0, 2))
            for l in ml:
                pts.append((g, l, abi.PATCH_SET_BALLOT, self.wb(nb), new_node, 0, 0))
                pts.append((g, l, abi.PATCH_RESIGN_COORD, 0, 0, 0, 0))
            pts.append((g, new_lane, abi.PATCH_INSTALL_COORD, self.wb(nb), new_node, self.ws(next_slot), 1))
            self.coord_idx[g] = self.members[g].index(new_node)
            self.promise_remote(g, (nb, new_node))  # phase 1 reached the remote members too
        if not pts:
            return
        p = np.zeros(len(pts), dtype=abi.patch_dtype)
        for i, t in enumerate(pts):
            p[i]["gid"], p[i]["lane"], p[i]["op"], p[i]["a"], p[i]["b"], p[i]["c"], p[i]["d"] = t
        for e in self.engines:
            e.patch(p)

    # ---- invariants ----------------------------------------------------------------------
    def check_safety(self):
        """Paxos safety as TESTPaxosApp asserts it: per replica, slots (unwrapped) are consecutive from 1 and
        any two replicas agree on the request of every slot both executed."""
        agreed = {}
        for lane in range(self.L):
            for g, seq in self.history[lane].items():
                slots = [s for s, _ in seq]
                assert slots == list(range(slots[0], slots[0] + len(slots))), f"gap at lane {lane} gid {g}: {slots}"
                for s, rid in seq:
                    k = (g, s)
                    if k in agreed:
                        assert agreed[k] == rid, f"replicas disagree on gid {g} slot {s}"
                    else:
                        agreed[k] = rid
        return len(agreed)

    def run(self, steps=60, rival=True, view_changes=True, stop_prob=0.01, check_every=10, fused_prob=0.0,
            round_prob=0.0, round_fn="round", prepares=False):
        for t in range(steps):
            if self.rng.random() < round_prob:
                self.step_round(frac=0.5, stop_prob=stop_prob, fn=round_fn)
            else:
                self.step_propose(frac=0.5, stop_prob=stop_prob)
            if rival and self.rng.random() < 0.3:
                self.inject_rival_accepts(int(self.rng.integers(1, 5)))
            if view_changes and self.rng.random() < 0.15:
                self.patch_view_change(int(self.rng.integers(1, 3)))
            if prepares and self.rng.random() < 0.3:
                self.step_prepares(int(self.rng.integers(1, 6)))
            order = self.rng.permutation(3)
            for o in order:
                if o == 0:
                    if self.rng.random() < fused_prob:
                        self.step_accepts_fused()
                    else:
                        self.step_accepts()
                elif o == 1:
                    self.step_replies()
                else:
                    self.step_decisions()
            if (t + 1) % check_every == 0:
                self.check_state()
        # drain
        for _ in range(6):
            self.step_accepts(p_deliver=1.0, p_dup=0, p_keep=0, lane_loss=0)
            self.step_replies(p_deliver=1.0, p_dup=0, p_keep=0)
            self.step_decisions(p_deliver=1.0, p_dup=0, p_keep=0, lane_loss=0)
        self.check_state()
        return self.check_safety()

    def close(self):
        for e in self.engines:
            e.close()
