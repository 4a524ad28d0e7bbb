"""Every entry point that logs, on one engine whose 64 KiB log ring wraps several times under log_backpressure.

After each call the host's mirror of the ring heads (what gpx_log_drain_async copies up to, and what the refusal test
reads) equals the head the kernels published.  And a call is refused with GPX_EAGAIN exactly when
head - released + 2 x bound > ring, with the bound each call passes to ring_fits:

  handle_accepts, accepts_device                  96 + 48 n + blob
  handle_accepts_fused                            160 + 80 n + blob
  handle_decisions, decisions_device, prepares    64 + 32 n
  round, round_phases, round_submit               192 + 80 n + pal + b1,  b1 = min(blob1_cap, 16 n + pal) when batching

The device round forms check no room: they are not refused, and the mirror follows them as well.
"""
import ctypes as C

import numpy as np
import pytest

from helpers import Engine, GpxErrorT, abi, group_descs, make_config, make_requests

pytestmark = pytest.mark.gpu

G, L, RING = 64, 3, 1 << 16
CFG = dict(max_groups=G, max_batch_recs=1024, max_batch_payload=1 << 14, log_ring_bytes=RING, log_backpressure=1)


def pal(pay):
    return (len(pay) + 15) & ~15


def round_bound(e, n, pay):
    b1 = min(((int(e.cfg.max_batch_payload) + 15) & ~15) + 16 * int(e.cfg.max_batch_recs), 16 * n + pal(pay))
    return 192 + 80 * n + pal(pay) + (b1 if e.cfg.batching_enabled else 0)


class Ring:
    """drains every lane after each call and releases on demand; checks the mirror against the device heads"""

    def __init__(self, e):
        self.e = e
        self.buf = np.zeros(RING, dtype=np.uint8)
        self.drained = [0] * L
        self.released = [0] * L
        self.refused = 0

    def check_mirror(self):
        for l in range(L):
            f, nb = self.e.log_drain_async(l, self.buf.ctypes.data, RING)
            self.e.log_drain_wait()
            assert f == self.drained[l]
            self.drained[l] = f + nb
            assert self.drained[l] == self.e.log_head(l), f"lane {l}: host mirror {self.drained[l]}"

    def release(self):
        for l in range(L):
            self.e.log_release(l, self.drained[l])
            self.released[l] = self.drained[l]

    def call(self, bound, fn):
        """fn() under ring_fits(bound); bound None: a call that checks no room"""
        if bound is None:
            out = fn()
            self.check_mirror()
            return out
        full = any(self.e.log_head(l) - self.released[l] + 2 * bound > RING for l in range(L))
        try:
            out = fn()
        except GpxErrorT as ex:
            assert ex.code == abi.GPX_EAGAIN and full, (ex.code, bound)
            self.refused += 1
            self.check_mirror()  # the refused call appended nothing
            self.release()
            assert all(self.e.log_head(l) - self.released[l] + 2 * bound <= RING for l in range(L))
            out = fn()
        else:
            assert not full, f"a call with bound {bound} was not refused"
        self.check_mirror()
        return out


def dev_round(e, fn, reqs, pay):
    import torch
    dev = torch.device("cuda", 0)
    n = len(reqs)
    d_reqs = torch.from_numpy(reqs.view(np.uint8).copy()).to(dev)
    d_pay = torch.from_numpy(np.concatenate([pay, np.zeros(16, np.uint8)])).to(dev)
    d_status = torch.zeros(n, dtype=torch.int32, device=dev)
    d_exec = torch.zeros(n * L * 24, dtype=torch.uint8, device=dev)
    bufs = abi.DevRoundBufs(d_reqs.data_ptr(), d_pay.data_ptr(), len(pay), n, d_status.data_ptr(), d_exec.data_ptr())
    torch.cuda.synchronize()
    e.L.check(e.L.fn(fn)(e.handle, C.byref(bufs), None))
    torch.cuda.synchronize()


def dev_accepts(e, acc, blob):
    """accepts_device -> host replies"""
    import torch
    dev = torch.device("cuda", 0)
    n = len(acc)
    d_acc = torch.from_numpy(acc.view(np.uint8).copy()).to(dev)
    d_blob = torch.from_numpy(np.concatenate([blob, np.zeros(16, np.uint8)])).to(dev)
    rep = torch.zeros(n * L * abi.reply_dtype.itemsize, dtype=torch.uint8, device=dev)
    extra = torch.zeros(4096 * abi.exec_dtype.itemsize, dtype=torch.uint8, device=dev)
    ctl = torch.zeros(8, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    e.L.check(e.L.fn("accepts_device")(e.handle, C.c_void_p(d_acc.data_ptr()), C.c_uint32(n),
                                       C.c_void_p(d_blob.data_ptr()), C.c_uint64(len(blob)), C.c_uint32(0), None, None,
                                       C.c_void_p(rep.data_ptr()), C.c_void_p(extra.data_ptr()), C.c_uint32(4096),
                                       C.c_void_p(ctl.data_ptr()), None))
    torch.cuda.synchronize()
    return rep.cpu().numpy().view(abi.reply_dtype)


def dev_decisions(e, dec):
    import torch
    dev = torch.device("cuda", 0)
    n = len(dec)
    d_dec = torch.from_numpy(dec.view(np.uint8).copy()).to(dev)
    ex = torch.zeros(n * L * abi.exec_dtype.itemsize, dtype=torch.uint8, device=dev)
    extra = torch.zeros(4096 * abi.exec_dtype.itemsize, dtype=torch.uint8, device=dev)
    ctl = torch.zeros(8, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    e.L.check(e.L.fn("decisions_device")(e.handle, C.c_void_p(d_dec.data_ptr()), C.c_uint32(n),
                                         C.c_void_p(ex.data_ptr()), C.c_void_p(extra.data_ptr()), C.c_uint32(4096),
                                         C.c_void_p(ctl.data_ptr()), None))
    torch.cuda.synchronize()


def test_host_mirror_and_refusal_threshold_of_every_logging_call(cuda_lib):
    e = Engine(cuda_lib, make_config(cuda_lib, **CFG))
    e.create_groups(group_descs(G))
    ring = Ring(e)
    gids = np.arange(G)
    rng = np.random.default_rng(12)
    kinds = ["accepts", "accepts_fused", "prepares", "round", "round_phases", "submit", "submit_compact",
             "round_device", "round_device_compact", "round_device_phases", "accepts_device"]
    step = 0
    for lap in range(6):
        for kind in kinds:
            sel = gids[rng.random(G) < 0.9]
            reqs, pay = make_requests(sel, payload_len=1 + step % 23, seed=12, round_no=step, entry_lane=step % L)
            step += 1
            if kind in ("accepts", "accepts_fused", "accepts_device"):
                acc, blob, _ = e.propose(reqs, pay)  # logs nothing
                n, nb = len(acc), len(blob)
                assert n > 0 and nb % 16 == 0
                if kind == "accepts_fused":
                    ring.call(160 + 80 * n + nb, lambda: e.handle_accepts_fused(acc, blob))
                    continue
                if kind == "accepts":
                    rep, _ = ring.call(96 + 48 * n + nb, lambda: e.handle_accepts(acc, blob))
                else:
                    rep = ring.call(96 + 48 * n + nb, lambda: dev_accepts(e, acc, blob))
                dec = e.handle_accept_replies(rep)  # logs nothing
                assert len(dec) > 0
                if kind == "accepts":
                    ring.call(64 + 32 * len(dec), lambda: e.handle_decisions(dec))
                else:
                    ring.call(64 + 32 * len(dec), lambda: dev_decisions(e, dec))
            elif kind == "prepares":  # a ballot below every group's: refused by the acceptors, logged all the same
                prep = np.zeros(len(sel), dtype=abi.decision_dtype)
                prep["gid"], prep["slot"] = sel, 1
                ring.call(64 + 32 * len(prep), lambda: e.handle_prepares(prep))
            elif kind in ("round", "round_phases"):
                ring.call(round_bound(e, len(reqs), pay), lambda: getattr(e, kind)(reqs, pay))
            elif kind.startswith("submit"):
                compact = kind == "submit_compact"
                t = ring.call(round_bound(e, len(reqs), pay), lambda: e.round_submit(reqs, pay, compact=compact))
                e.round_wait(t)
                ring.check_mirror()
            else:
                ring.call(None, lambda: dev_round(e, kind, reqs, pay))
    assert ring.refused >= 5, "the ring was sized to fill up several times"
    assert all(e.log_head(l) > 4 * RING for l in range(L)), "the ring wraps several times"
    e.close()
