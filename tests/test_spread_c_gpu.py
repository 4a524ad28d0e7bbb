"""GPU parity of SPREAD placement behind the C ABI (gpx_spread_*: include/gpx.h, gigapaxos_b200/csrc/gpx_spread.cuh).

N single-lane CUDA engines -- in `local` mode all on one GPU, the exchange being device copies; the NCCL mode of the
multi-GPU run moves the very same buckets -- against ONE oracle engine that hosts all N nodes as lanes and is driven
phase by phase.  Per node: request status, the EXEC sequence, every state row, the non-VOID log images + logged payload
bytes and the counters must be identical (integer / byte work: bit-exact).

Reference behaviour: replica j of a group on node (home + j) mod N, coordinator PISM.roundRobinCoordinator :2251-2256,
unicast fan-out paxosutil/PaxosMessenger.java:175-182.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import Engine, abi, canon, make_config, make_requests
from gigapaxos_b200.spread import Spread, coordinator_of, members_of, spread_caps, spread_config

pytestmark = pytest.mark.gpu

NODE0 = 100


def make_groups(N, G, R):
    node_ids = [NODE0 + i for i in range(N)]
    descs = np.zeros(G, dtype=abi.group_desc_dtype)
    descs["gid"] = np.arange(G)
    descs["n_members"] = R
    descs["init_mode"] = abi.INIT_BATCH
    coord = np.zeros(G, dtype=np.int64)
    member_of = np.zeros((G, N), dtype=bool)
    for g in range(G):
        nm = f"NoopPaxosApp{g}"
        mem = [node_ids[m] for m in members_of(nm, N, R)]
        descs["name_hash"][g] = abi.java_string_hash(nm)
        descs["members"][g, :R] = mem
        coord[g] = coordinator_of(nm, mem) - NODE0
        member_of[g, [m - NODE0 for m in mem]] = True
    return node_ids, descs, coord, member_of


class Cluster:
    """N CUDA nodes + the spread handle + per-node device buffers"""

    def __init__(self, cuda_lib, N, G, R, P, graph=False, slots=1, p2p=False, **cfg):
        import torch
        self.torch = torch
        self.N, self.G = N, G
        self.node_ids, self.descs, self.coord, self.member_of = make_groups(N, G, R)
        self.dev = torch.device("cuda", 0)
        self.engines = []
        for i in range(N):
            c = make_config(cuda_lib, max_groups=G, n_lanes=1, lane_node=[self.node_ids[i]], max_group_size=R,
                            max_batch_recs=4 * G, max_batch_payload=1 << 22, **cfg)
            e = Engine(cuda_lib, c)
            e.create_groups(self.descs[self.member_of[:, i]])
            self.engines.append(e)
        cap = spread_caps(self.coord, self.member_of, slots_per_round=slots, slack=3)
        # a batched slot carries 16 B per request + the bodies
        self.scfg = spread_config(self.node_ids, cap, blob_per_rec=4 * (16 + ((P + 15) // 16) * 16), max_reqs=4 * G,
                                  graph=graph, p2p=p2p)
        self.sp = Spread(cuda_lib, self.engines, self.scfg)
        self.stream = torch.cuda.Stream(device=self.dev)
        self.ctl = [torch.zeros(8, dtype=torch.int32, device=self.dev) for _ in range(N)]
        self.exec = [torch.zeros(max(p.vtotal, 1) * 24, dtype=torch.uint8, device=self.dev) for p in self.sp.plans]
        self.extra = [torch.zeros(4096 * 24, dtype=torch.uint8, device=self.dev) for _ in range(N)]
        self.status = [torch.zeros(4 * G, dtype=torch.int32, device=self.dev) for _ in range(N)]
        self.keep = []
        self.drain = np.empty(int(self.engines[0].cfg.log_ring_bytes), dtype=np.uint8)

    def round(self, reqs, pay, fixed=None):
        """split the global batch by coordinator node and run one spread round; returns per node (status, exec)"""
        torch = self.torch
        gids = reqs["gid"]
        ios, index = [], {}
        self.keep = []
        for i in range(self.N):
            sel = np.nonzero(self.coord[gids] == i)[0]
            index[i] = sel
            io = abi.SpreadIO()
            io.n = len(sel)
            if len(sel):
                rq = reqs[sel].copy()
                rq["flags"] &= ~np.uint32(0xF00)  # single-lane node: entry lane 0
                stride = ((rq["payload_len"] + 15) // 16) * 16
                offs = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint32)
                buf = np.zeros(int(stride.sum()) + 16, dtype=np.uint8)
                for k in range(len(rq)):
                    o, ln = int(reqs["payload_off"][sel[k]]), int(rq["payload_len"][k])
                    buf[offs[k]: offs[k] + ln] = pay[o: o + ln]
                rq["payload_off"] = offs
                if fixed is not None and i in fixed:  # reuse device buffers (CUDA-graph replay needs equal pointers)
                    dr, dp = fixed[i]
                    dr[: rq.nbytes].copy_(torch.from_numpy(rq.view(np.uint8).copy()))
                    dp[: buf.size].copy_(torch.from_numpy(buf))
                else:
                    dr = torch.from_numpy(rq.view(np.uint8).copy()).to(self.dev)
                    dp = torch.from_numpy(buf).to(self.dev)
                self.keep += [dr, dp]
                io.reqs, io.payload, io.payload_bytes = dr.data_ptr(), dp.data_ptr(), int(stride.sum())
            io.status = self.status[i].data_ptr()
            io.exec = self.exec[i].data_ptr()
            io.extra, io.extra_cap = self.extra[i].data_ptr(), 4096
            io.ctl = self.ctl[i].data_ptr()
            ios.append(io)
        torch.cuda.synchronize()
        self.sp.round(ios, self.stream.cuda_stream)
        torch.cuda.synchronize()
        out = {}
        for i in range(self.N):
            ex = self.exec[i].cpu().numpy().view(abi.exec_dtype)[: self.sp.plans[i].vtotal]
            out[i] = (self.status[i].cpu().numpy()[: len(index[i])], ex, self.ctl[i].cpu().numpy().copy())
        return out, index

    def close(self):
        self.sp.close()
        for e in self.engines:
            e.close()


def oracle_round(eo, reqs, pay):
    acc, blob, status = eo.propose(reqs, pay)
    replies, x1 = eo.handle_accepts(acc, blob, extra_cap=4 * len(acc) + 16)
    dec = eo.handle_accept_replies(replies)
    ex, x2 = eo.handle_decisions(dec, extra_cap=4 * len(acc) + 16)
    return status, ex, np.concatenate([x1, x2])


def by_gid(recs):
    r = recs[(recs["flags"] & abi.F_VOID) == 0]
    return r[np.argsort(r["gid"], kind="stable")]


def compare_state_logs_counters(eo, cl):
    for i, e in enumerate(cl.engines):
        g = np.nonzero(cl.member_of[:, i])[0]
        ro, rg = eo.dump_rows(g, i), e.dump_rows(g, 0)
        for f in ro.dtype.names:
            if f != "lane":
                assert np.array_equal(ro[f], rg[f]), f"node {i} row field {f}"
    for i, e in enumerate(cl.engines):
        so_ = [s for s in abi.parse_log(eo.log_read(i)) if len(canon(s[1])) > 0]
        sg_ = [s for s in abi.parse_log(e.log_read(0)) if len(canon(s[1])) > 0]
        assert len(so_) == len(sg_) > 0, (i, len(so_), len(sg_))
        for (ho, io_, po, _), (hg, ig, pg, _) in zip(so_, sg_):
            assert int(ho["type"]) == int(hg["type"])
            co, cg = canon(io_), canon(ig)
            assert len(co) == len(cg)
            for f in co.dtype.names:
                if f not in ("payload_off", "dst_mask"):
                    assert np.array_equal(co[f], cg[f]), f"node {i} log image {f}"
            if int(ho["rec_bytes"]) == 48:
                for a, b in zip(co, cg):
                    ao, bo, ln = int(a["payload_off"]), int(b["payload_off"]), int(a["payload_len"])
                    x, y = po[ao: ao + ln].copy(), pg[bo: bo + ln].copy()
                    nreq = int(a["nreq"])
                    if nreq > 1:  # batched blob: the per-request flags carry the ENTRY LANE, a per-engine notion
                        for t in (x, y):
                            t[: 16 * nreq].view(abi.batch_ent_dtype)["flags"] &= ~np.uint32(0xF00)
                    assert np.array_equal(x, y), ("log payload", i, int(a["gid"]), nreq, ln)
    co = eo.counters()
    tot = {k: 0 for k in co}
    for e in cl.engines:
        for k, v in e.counters().items():
            tot[k] += v
    for k in ("accepts_handled", "accepts_acked", "accepts_logged", "replies_handled", "decisions_made",
              "decisions_handled", "executed", "checkpoints_due", "proposals", "requests_batched"):
        assert co[k] == tot[k], (k, co[k], tot[k])


def check_round(cl, res, index, so, xo):
    for i in range(cl.N):
        st, ex, ctl = res[i]
        if len(index[i]):
            assert np.array_equal(st, so[index[i]]), f"status node {i}"
        assert ctl[2] == 0, "no extra executions expected"
        lanes_o = (xo["flags"] >> 12) & 0xF
        want, got = by_gid(xo[lanes_o == i]), by_gid(ex)
        assert len(want) == len(got), (i, len(want), len(got), ctl.tolist())
        for f in ("gid", "slot", "req_id"):
            assert np.array_equal(want[f], got[f]), f"node {i} exec {f}"
        assert np.array_equal(want["flags"] & ~np.uint32(0xF000), got["flags"] & ~np.uint32(0xF000))
    for i, e in enumerate(cl.engines):  # the host's mirror of the ring head (what a drain copies up to) follows the kernels
        f, nb = e.log_drain_async(0, cl.drain.ctypes.data, len(cl.drain))
        e.log_drain_wait()
        assert f + nb == e.log_head(0), f"node {i}: ring head mirror"


@pytest.mark.parametrize("N,G,P,graph,p2p", [(4, 600, 1, False, False), (3, 200, 40, False, False), (5, 333, 17, False, False),
                                             (8, 900, 5, False, False), (4, 600, 17, True, False), (5, 100, 17, False, False),
                                             (4, 600, 1, False, True), (8, 900, 5, False, True), (4, 600, 17, True, True)])
def test_spread_c_round_parity(oracle_lib, cuda_lib, N, G, P, graph, p2p):
    """p2p: the peer-memory transport (send buckets ARE the peers' receive buckets, k_sp_signal / k_sp_wait); between
    engines of one process the peers' arenas are plain device pointers, between processes CUDA IPC mappings"""
    R = 3
    cl = Cluster(cuda_lib, N, G, R, P, graph=graph, p2p=p2p, checkpoint_interval=3)
    eo = Engine(oracle_lib, make_config(oracle_lib, max_groups=G, n_lanes=N, lane_node=cl.node_ids, max_group_size=R,
                                        max_batch_recs=4 * G, max_batch_payload=1 << 22, checkpoint_interval=3))
    eo.create_groups(cl.descs)
    rng = np.random.default_rng(5)
    n_exec = 0
    fixed = None
    if graph:  # equal io blocks (pointers, n, payload bytes) from round to round: the captured graph is REPLAYED
        import torch
        fixed = {i: (torch.zeros(4 * G * 32, dtype=torch.uint8, device=cl.dev),
                     torch.zeros(4 * G * 64 + 64, dtype=torch.uint8, device=cl.dev)) for i in range(N)}
        counts0 = rng.choice([0, 1, 1, 1, 2, 3], size=G)
    for r in range(6):
        counts = rng.choice([0, 1, 1, 1, 2, 3], size=G)  # several requests of a group -> one batched slot; some idle
        if graph:
            counts = counts0.copy()
        elif r == 4:
            counts[:] = 0
            counts[:: max(G // 7, 1)] = 1  # a sparse round: most buckets nearly empty
        gids = np.repeat(np.arange(G), counts)
        lens = rng.integers(1, P + 1, size=len(gids)) if not graph else np.full(len(gids), P)
        reqs, pay = make_requests(gids, payload_len=lens, seed=31, round_no=r)
        reqs["flags"] = (cl.coord[gids].astype(np.uint32) << 8)  # oracle: entry lane = the coordinator's lane
        reqs["entry_node"] = NODE0 + cl.coord[gids]
        so, xo, extra_o = oracle_round(eo, reqs, pay)
        assert len(extra_o) == 0
        res, index = cl.round(reqs, pay, fixed)
        check_round(cl, res, index, so, xo)
        n_exec += sum(len(by_gid(res[i][1])) for i in range(N))
    assert n_exec > 0
    for k in range(N):
        assert cl.sp.dropped(k) == 0
    compare_state_logs_counters(eo, cl)
    cl.close()
    eo.close()


def test_spread_c_five_replicas_and_stops(oracle_lib, cuda_lib):
    """R = 5 over 6 nodes, STOP requests inside the stream (epoch ends: PISM.handleCommittedRequest stop path)"""
    N, G, R, P = 6, 240, 5, 9
    cl = Cluster(cuda_lib, N, G, R, P, checkpoint_interval=4)
    eo = Engine(oracle_lib, make_config(oracle_lib, max_groups=G, n_lanes=N, lane_node=cl.node_ids, max_group_size=R,
                                        max_batch_recs=4 * G, max_batch_payload=1 << 22, checkpoint_interval=4))
    eo.create_groups(cl.descs)
    rng = np.random.default_rng(9)
    for r in range(5):
        counts = rng.choice([0, 1, 1, 2], size=G)
        gids = np.repeat(np.arange(G), counts)
        stop = (rng.random(len(gids)) < 0.03) if r >= 2 else None
        reqs, pay = make_requests(gids, payload_len=rng.integers(1, P + 1, size=len(gids)), seed=77, round_no=r,
                                  stop_mask=stop)
        reqs["flags"] |= (cl.coord[gids].astype(np.uint32) << 8)
        reqs["entry_node"] = NODE0 + cl.coord[gids]
        so, xo, extra_o = oracle_round(eo, reqs, pay)
        assert len(extra_o) == 0
        res, index = cl.round(reqs, pay)
        check_round(cl, res, index, so, xo)
    compare_state_logs_counters(eo, cl)
    cl.close()
    eo.close()


# ---- one process per GPU over NCCL inside libgpx (needs >= 3 GPUs: skipped on single-GPU boxes) -----------------
def _nccl_worker(rank, world, port, q, G, rounds, graph, p2p=False):
    import os
    import traceback
    import torch
    import torch.distributed as dist
    try:
        os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
        os.environ.setdefault("NCCL_DEBUG", "WARN")
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("gloo", rank=rank, world_size=world)  # only to hand the NCCL unique id around
        import gigapaxos_b200
        from helpers import oracle_library
        R, P = 3, 24
        node_ids, descs, coord, member_of = make_groups(world, G, R)
        lib = gigapaxos_b200.load_library()
        e = Engine(lib, make_config(lib, device=rank, max_groups=G, n_lanes=1, lane_node=[node_ids[rank]],
                                    max_group_size=R, max_batch_recs=4 * G, max_batch_payload=1 << 22,
                                    checkpoint_interval=3))
        e.create_groups(descs[member_of[:, rank]])
        scfg = spread_config(node_ids, spread_caps(coord, member_of, slack=2), blob_per_rec=4 * (16 + 32),
                             max_reqs=4 * G, graph=graph, p2p=p2p)
        ids = [Spread.unique_id(lib) if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        sp = Spread(lib, [e], scfg, rank=rank, unique_id=ids[0])
        plan = sp.plans[0]
        olib = oracle_library()
        ref = Engine(olib, make_config(olib, max_groups=G, n_lanes=world, lane_node=node_ids, max_group_size=R,
                                       max_batch_recs=4 * G, max_batch_payload=1 << 22, checkpoint_interval=3))
        ref.create_groups(descs)
        stream = torch.cuda.Stream(device=dev)
        ctl = torch.zeros(8, dtype=torch.int32, device=dev)
        ex = torch.zeros(plan.vtotal * 24, dtype=torch.uint8, device=dev)
        extra = torch.zeros(1024 * 24, dtype=torch.uint8, device=dev)
        status = torch.zeros(4 * G, dtype=torch.int32, device=dev)
        d_reqs = torch.zeros(4 * G * 32, dtype=torch.uint8, device=dev)
        d_pay = torch.zeros(4 * G * 48 + 64, dtype=torch.uint8, device=dev)
        n_exec = 0
        rng = np.random.default_rng(100)  # same stream of random numbers on every rank
        for r in range(rounds):
            counts = rng.choice([0, 1, 1, 2, 3], size=G)
            gids = np.repeat(np.arange(G), counts)
            lens = rng.integers(1, P + 1, size=len(gids))
            reqs, pay = make_requests(gids, payload_len=lens, seed=77, round_no=r)
            reqs["flags"] = coord[gids].astype(np.uint32) << 8
            reqs["entry_node"] = NODE0 + coord[gids]
            so, xo, _ = oracle_round(ref, reqs, pay)
            sel = np.nonzero(coord[gids] == rank)[0]
            io = abi.SpreadIO()
            io.n = len(sel)
            if len(sel):
                rq = reqs[sel].copy()
                rq["flags"] &= ~np.uint32(0xF00)
                stride = ((rq["payload_len"] + 15) // 16) * 16
                offs = np.concatenate([[0], np.cumsum(stride)[:-1]]).astype(np.uint32)
                buf = np.zeros(int(stride.sum()) + 16, dtype=np.uint8)
                for k in range(len(rq)):
                    o, ln = int(reqs["payload_off"][sel[k]]), int(rq["payload_len"][k])
                    buf[offs[k]: offs[k] + ln] = pay[o: o + ln]
                rq["payload_off"] = offs
                d_reqs[: rq.nbytes].copy_(torch.from_numpy(rq.view(np.uint8).copy()))
                d_pay[: buf.size].copy_(torch.from_numpy(buf))
                io.reqs, io.payload, io.payload_bytes = d_reqs.data_ptr(), d_pay.data_ptr(), int(stride.sum())
            io.status, io.exec, io.extra, io.extra_cap, io.ctl = (status.data_ptr(), ex.data_ptr(), extra.data_ptr(), 1024,
                                                                  ctl.data_ptr())
            torch.cuda.synchronize()
            sp.round([io], stream.cuda_stream)
            torch.cuda.synchronize()
            if len(sel):
                assert np.array_equal(status.cpu().numpy()[: len(sel)], so[sel])
            got = by_gid(ex.cpu().numpy().view(abi.exec_dtype)[: plan.vtotal])
            want = by_gid(xo[((xo["flags"] >> 12) & 0xF) == rank])
            assert len(got) == len(want), (len(got), len(want))
            for f in ("gid", "slot", "req_id"):
                assert np.array_equal(got[f], want[f]), f
            n_exec += len(got)
        assert sp.dropped(0) == 0
        g = np.nonzero(member_of[:, rank])[0]
        ro, rg = ref.dump_rows(g, rank), e.dump_rows(g, 0)
        for f in ro.dtype.names:
            if f != "lane":
                assert np.array_equal(ro[f], rg[f]), f
        dist.barrier()
        q.put((rank, "ok", n_exec))
        sp.close()
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        q.put((rank, "fail: " + traceback.format_exc(), 0))
        raise


# (graph, p2p) = (True, True) is exercised by `bench.py --gpus 4 --p2p` (replay of four captured rounds, counters
# asserted) and by the local-mode parity test above; as a multi-process parity test -- a NEW graph captured every round,
# over IPC mappings -- it timed out once on the 4-GPU box and is left out of the matrix until that is understood.
@pytest.mark.parametrize("graph,p2p", [(False, False), (True, False), (False, True)])
def test_spread_c_over_nccl(graph, p2p):
    import torch
    import torch.multiprocessing as mp
    from test_spread_gloo import free_port
    world = min(torch.cuda.device_count(), 8)
    if world < 3:
        pytest.skip("spread placement over NCCL needs >= 3 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_nccl_worker, args=(r, world, port, q, 500, 5, graph, p2p)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, status, n_exec in res:
        assert status == "ok", f"rank {rank}: {status}"
        assert n_exec > 0
