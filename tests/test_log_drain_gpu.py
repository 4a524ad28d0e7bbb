"""Log ring tail, back-pressure and asynchronous drain (VERDICT r1 item 4).

AbstractPaxosLogger.logAndMessage :157 / BatchedLogger :691-716 log THEN message, SQLPaxosLogger.journal :965-1036 appends
to a file: a ring position may only be reused once its bytes are durable elsewhere.  With gpx_config.log_backpressure a
call that could overwrite unreleased bytes is refused with GPX_EAGAIN before it does anything; the drain copies on its
own stream while rounds continue.  The drained byte stream, re-parsed, must equal the oracle's (unbounded) log segment
by segment -- i.e. no undrained byte was ever overwritten -- across many ring wraps.
"""
import numpy as np
import pytest

from helpers import Engine, GpxErrorT, abi, canon, exec_by_lane, group_descs, make_config, make_requests

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["round", "round_phases"])
def test_backpressure_and_drain_keep_every_byte(oracle_lib, cuda_lib, mode):
    import torch
    G, R, ring = 300, 3, 1 << 17  # one round appends ~40 KB per lane: a 128 KiB ring fills after a few rounds
    kw = dict(max_groups=G, max_batch_recs=1024, max_batch_payload=1 << 16, log_ring_bytes=ring)
    eo = Engine(oracle_lib, make_config(oracle_lib, **kw))
    eg = Engine(cuda_lib, make_config(cuda_lib, log_backpressure=1, **kw))
    d = group_descs(G)
    eo.create_groups(d)
    eg.create_groups(d)
    pinned = [torch.zeros(ring, dtype=torch.uint8).pin_memory() for _ in range(R)]
    drained = [[] for _ in range(R)]
    refused = rounds_done = 0
    gids = np.arange(G)
    r = 0
    while rounds_done < 40:
        reqs, pay = make_requests(gids, payload_len=1 + r % 20, seed=5, round_no=r, entry_lane=r % R)
        try:
            sg, xg, _ = getattr(eg, mode)(reqs, pay)
        except GpxErrorT as ex:
            assert ex.code == abi.GPX_EAGAIN
            refused += 1
            # drain everything that is there, asynchronously, then release it
            upto = []
            for l in range(R):
                f, nb = eg.log_drain_async(l, pinned[l].data_ptr(), ring)
                upto.append((f, nb))
            eg.log_drain_wait()
            for l, (f, nb) in enumerate(upto):
                assert nb > 0
                drained[l].append((f, pinned[l].numpy()[:nb].copy()))
                eg.log_release(l, f + nb)
            continue  # the refused call did nothing: repeat it
        so, xo, _ = getattr(eo, mode)(reqs, pay)
        assert np.array_equal(so, sg)
        for a, b in zip(exec_by_lane(xo, R), exec_by_lane(xg, R)):
            for f in ("gid", "slot", "req_id", "flags"):
                assert np.array_equal(a[f], b[f])
        rounds_done += 1
        r += 1
    assert refused >= 5, "the ring was sized to fill up several times"
    for l in range(R):  # the tail
        f, nb = eg.log_drain_async(l, pinned[l].data_ptr(), ring)
        eg.log_drain_wait()
        if nb:
            drained[l].append((f, pinned[l].numpy()[:nb].copy()))
    for l in range(R):
        assert all(drained[l][k][0] + len(drained[l][k][1]) == drained[l][k + 1][0] for k in range(len(drained[l]) - 1))
        assert drained[l][-1][0] + len(drained[l][-1][1]) > 8 * ring, "many wraps"
        buf = np.concatenate([c[1] for c in drained[l]])
        sg_ = [(h, im, p) for (h, im, p, _) in abi.parse_log(buf, ring, drained[l][0][0])]
        so_ = [(h, im, p) for (h, im, p, _) in abi.parse_log(eo.log_read(l))]
        assert len(sg_) == len(so_) > 0, (l, len(sg_), len(so_))
        for (ho, io_, po), (hg, ig, pg) in zip(so_, sg_):
            for f in ("type", "lane", "payload_bytes", "seq", "rec_bytes"):
                assert int(ho[f]) == int(hg[f]), f"lane {l} seg hdr {f}"
            co, cg = canon(io_), canon(ig)
            assert len(co) == len(cg)
            for f in co.dtype.names:
                if f != "payload_off":
                    assert np.array_equal(co[f], cg[f]), f"lane {l} image {f}"
            if int(ho["rec_bytes"]) == 48:
                for a, b in zip(co, cg):
                    x, y, n = int(a["payload_off"]), int(b["payload_off"]), int(a["payload_len"])
                    assert np.array_equal(po[x: x + n], pg[y: y + n])
    eo.close()
    eg.close()


def test_release_beyond_drained_is_refused(cuda_lib):
    eg = Engine(cuda_lib, make_config(cuda_lib, max_groups=16, log_backpressure=1))
    with pytest.raises(GpxErrorT):
        eg.log_release(0, 4096)
    eg.close()
