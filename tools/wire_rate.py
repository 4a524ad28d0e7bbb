"""Packets/s and records/s of the phase-2 wire codec: the device calls (gpx_wire_decode_batch, gpx_wire_encode_*) at
100 K and 1 M groups with one packet per group per round, and the host codec (gpx_wire_decode_accept /
gpx_wire_encode_batched_commit, one packet per call) on one thread and on every host thread.

Device numbers come two ways: the wall time of the C call, which includes the host->device and device->host copies
and ends in a device synchronise; and the kernel time alone, the sum of the CUDA kernels torch.profiler records during
a separate pass.  The host codec runs in a small C program built into a temporary directory and linked against
libgpx.so, so no Python sits in its loop.  The card, its power limit and its SM clock are read in the same run.

`acceptor_chain` times an acceptor's whole phase-2 path (decode the ACCEPTs, handle them, encode the replies) two ways:
through the device-buffer forms with one upload of the packets and one download of the replies, and through the
host-buffer calls (see acceptor_chain).

    python tools/wire_rate.py [--groups 100000 1000000] [--reps 5] [--out FILE.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HOST_BENCH = r"""
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include "gpx.h"
#include "gpx_wire.h"
static const uint8_t* g_bytes; static const gpx_wire_ref* g_refs; static uint32_t g_n; static int g_mode;
static int32_t g_group[3] = {100, 101, 102};
static void* run(void* arg) {
  const uintptr_t t = (uintptr_t)arg; /* thread index << 8 | thread count */
  uint32_t lo = (uint32_t)(((uint64_t)g_n * (t >> 8)) / (t & 0xff)), hi = (uint32_t)(((uint64_t)g_n * ((t >> 8) + 1)) / (t & 0xff));
  gpx_wire_accept_view v; uint8_t out[512]; long sink = 0;
  for (uint32_t i = lo; i < hi; i++) {
    if (g_mode == 0) { if (gpx_wire_decode_accept(g_bytes + g_refs[i].off, g_refs[i].len, &v) == 0) sink += v.slot; }
    else { int32_t s = (int32_t)i; sink += (long)gpx_wire_encode_batched_commit((const char*)g_bytes + g_refs[i].off + 13,
             g_bytes[g_refs[i].off + 12], 0, 1, 100, 0, 1, &s, 3, g_group, out, sizeof out); }
  }
  return (void*)sink;
}
int main(int argc, char** argv) {
  FILE* f = fopen(argv[1], "rb"); fseek(f, 0, SEEK_END); long sz = ftell(f); fseek(f, 0, SEEK_SET);
  uint8_t* b = (uint8_t*)malloc(sz); if (fread(b, 1, sz, f) != (size_t)sz) return 1; fclose(f);
  f = fopen(argv[2], "rb"); fseek(f, 0, SEEK_END); long rs = ftell(f); fseek(f, 0, SEEK_SET);
  gpx_wire_ref* r = (gpx_wire_ref*)malloc(rs); if (fread(r, 1, rs, f) != (size_t)rs) return 1; fclose(f);
  g_bytes = b; g_refs = r; g_n = (uint32_t)(rs / sizeof(gpx_wire_ref)); g_mode = atoi(argv[3]);
  int T = atoi(argv[4]); pthread_t th[256]; struct timespec a, c;
  clock_gettime(CLOCK_MONOTONIC, &a);
  for (int t = 0; t < T; t++) pthread_create(&th[t], 0, run, (void*)(uintptr_t)(((uintptr_t)t << 8) | (uintptr_t)T));
  for (int t = 0; t < T; t++) pthread_join(th[t], 0);
  clock_gettime(CLOCK_MONOTONIC, &c);
  printf("%.9f\n", (c.tv_sec - a.tv_sec) + 1e-9 * (c.tv_nsec - a.tv_nsec));
  return 0;
}
"""


def card_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # pragma: no cover
        out = f"unavailable: {ex}"
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def kernel_ms(fn):
    """sum of CUDA kernel time during one call of fn (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = 0.0
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and not ev.name.startswith("Memcpy") and not ev.name.startswith("Memset"):
            tot += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return tot / 1000.0


def with_round(arena, refs, slot, bnum):
    """the ACCEPT packets of `arena` with their slot and ballot number rewritten (big-endian, in the 22-byte trailer
    slot, bnum, bcoord, recovery, median, noCoalesce, sender of AcceptPacket)"""
    a = arena.copy()
    end = refs["off"].astype(np.int64) + refs["len"].astype(np.int64)
    for at, v in ((end - 22, slot), (end - 18, bnum)):
        for k in range(4):
            a[at + k] = (v >> (24 - 8 * k)) & 0xFF
    return a


def acceptor_chain(lib, G, arena, refs, reps):
    """An acceptor's whole phase-2 path for one ACCEPT per group, addressed to a node-101 engine: decode, handle, encode
    the replies.  Every repetition is a fresh round (slot r, ballot (1, 100), above every group's initial ballot) made
    before timing, so each does the same protocol work; `reps` + 2 rounds must fit the window of 8.

    * device leg: pinned host arena -> one upload -> gpx_wire_decode_batch_device -> gpx_accepts_device ->
      gpx_wire_encode_replies_device -> one download of the reply packets;
    * host-buffer leg: gpx_wire_decode_batch -> gpx_handle_accepts -> gpx_wire_encode_replies as bare C calls, on a
      second engine in the same state.
    The legs alternate; wall time to a device synchronise, best of `reps`, then the kernel-only sum of one more round
    of each leg under torch.profiler."""
    import ctypes as C

    import torch

    from gigapaxos_b200 import abi, wire
    from helpers import Engine, group_descs_fast, make_config

    assert reps + 2 <= 8, "every round takes a slot of the window"
    ring = 1 << 16
    while ring < 2 * (96 + 64 * G):
        ring <<= 1
    engines = []
    for _ in range(2):
        e = Engine(lib, make_config(lib, max_groups=G, n_lanes=1, lane_node=[101], window=8, max_batch_recs=G,
                                    max_batch_payload=16 * G, log_ring_bytes=ring))
        e.create_groups(group_descs_fast(G, members=(100, 101, 102)))
        wire.set_group_names(e, np.arange(G, dtype=np.uint32), [f"NoopPaxosApp{i}" for i in range(G)])
        engines.append(e)
    ed, eh = engines
    rounds = [with_round(arena, refs, r, 1) for r in range(reps + 2)]
    fn = lib.fn
    st = wire.stream_handle()
    ptr = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    # device leg: pinned staging and device buffers made once
    h_refs = torch.from_numpy(refs.view(np.uint8).reshape(G, 16).copy()).pin_memory()
    h_arenas = [torch.from_numpy(a).pin_memory() for a in rounds]
    d_arena = torch.empty(len(arena), dtype=torch.uint8, device="cuda")
    d_refs = torch.empty((G, 16), dtype=torch.uint8, device="cuda")
    ctl = torch.zeros(8, dtype=torch.int32, device="cuda")
    d_rep = torch.empty((G, 32), dtype=torch.uint8, device="cuda")
    d_extra = torch.empty((4096, 24), dtype=torch.uint8, device="cuda")
    h_out = torch.empty(128 * G, dtype=torch.uint8).pin_memory()
    h_out_refs = torch.empty((G, 16), dtype=torch.uint8).pin_memory()
    caps = {"dec": (G, 16 * G, 1, 1), "enc": (128 * G, G)}

    def device_leg(r):
        d_arena.copy_(h_arenas[r], non_blocking=True)
        d_refs.copy_(h_refs, non_blocking=True)
        d = wire.decode_batch_device(ed, d_arena, d_refs, caps["dec"])
        ctl.zero_()
        na = d.sizes[0]
        lib.check(fn("accepts_device")(ed.handle, ptr(d.accepts), C.c_uint32(na), ptr(d.blob), C.c_uint64(d.sizes[1]),
                                       C.c_uint32(0), None, None, ptr(d_rep), ptr(d_extra), C.c_uint32(4096), ptr(ctl),
                                       st))
        enc = wire.encode_replies_device(ed, d_rep, na, caps["enc"])
        caps["dec"], caps["enc"] = d.sizes, enc.sizes
        h_out[: enc.sizes[0]].copy_(enc.out, non_blocking=True)
        h_out_refs[: enc.sizes[1]].copy_(enc.refs, non_blocking=True)
        torch.cuda.synchronize()
        return enc.sizes

    # host-buffer leg: numpy buffers made once
    status = np.zeros(G, np.int32)
    acc = np.zeros(G, abi.accept_dtype)
    blob = np.zeros(16 * G, np.uint8)
    z = np.zeros(1, abi.reply_dtype)
    rep = np.zeros(G, abi.reply_dtype)
    extra = np.zeros(4096, abi.exec_dtype)
    rst = np.zeros(G, np.uint8)
    out = np.zeros(128 * G, np.uint8)
    out_refs = np.zeros(G, abi.wire_ref_dtype)

    def host_leg(r):
        a = rounds[r]
        sz = [C.c_uint32(G), C.c_uint64(len(blob)), C.c_uint32(0), C.c_uint32(0)]
        lib.check(fn("wire_decode_batch")(eh.handle, C.c_uint32(G), abi._ptr(a), C.c_uint64(len(a)), abi._ptr(refs),
                                          abi._ptr(status), abi._ptr(acc), C.byref(sz[0]), abi._ptr(blob),
                                          C.byref(sz[1]), abi._ptr(z), C.byref(sz[2]), abi._ptr(z), C.byref(sz[3])))
        nx = C.c_uint32(0)
        lib.check(fn("handle_accepts")(eh.handle, sz[0], abi._ptr(acc), abi._ptr(blob), C.c_uint64(sz[1].value),
                                       abi._ptr(rep), abi._ptr(extra), C.c_uint32(len(extra)), C.byref(nx)))
        nb, nr = C.c_uint64(len(out)), C.c_uint32(G)
        lib.check(fn("wire_encode_replies")(eh.handle, sz[0], abi._ptr(rep), abi._ptr(rst), abi._ptr(out),
                                            C.byref(nb), abi._ptr(out_refs), C.byref(nr)))
        return nb.value, nr.value

    walls = {"device": [], "host_buffer": []}
    sizes = {}
    for r in range(reps + 1):  # round 0 warms both legs up
        for leg, run in (("device", device_leg), ("host_buffer", host_leg)):
            t = time.perf_counter()
            sizes[leg] = run(r)
            if r:
                walls[leg].append(time.perf_counter() - t)
    # both legs wrote the same reply packets
    assert tuple(sizes["device"]) == tuple(sizes["host_buffer"])
    nb, nr = sizes["device"]
    assert nr == G, "every ACCEPT is accepted and its reply is encoded"
    assert bytes(h_out[:nb].numpy()) == out[:nb].tobytes() and bytes(h_out_refs[:nr].numpy()) == out_refs[:nr].tobytes()
    res = {"packets": G, "reply_packets": int(nr), "reply_bytes": int(nb), "upload_bytes": int(len(arena) + 16 * G),
           "log_ring_bytes": ring}
    for leg, run in (("device", device_leg), ("host_buffer", host_leg)):
        w = min(walls[leg])
        res[leg] = {"wall_s_min": w, "packets_per_s_wall": G / w,
                    "kernel_ms": kernel_ms(lambda: run(reps + 1))}
        res[leg]["packets_per_s_kernels"] = G / (res[leg]["kernel_ms"] / 1000.0)
    for e in engines:
        e.close()
    return res


def coordinator_chain(lib, G, reps):
    """node 100 as the coordinator of G groups {100, 101, 102}, one client REQUEST per group it coordinates per round.
    Device leg: one upload of the request arena, decode_requests_device -> propose_device_heads ->
    encode_accepts_device, one download of the ACCEPT arena.  Host leg: the same requests through gpx_propose (host
    records) and the per-packet host encoder (wire.encode_accept, one call per ACCEPT).  The legs alternate on two
    engines in the same state and must write the same ACCEPT packets."""
    import ctypes as C

    import torch

    from gigapaxos_b200 import abi, wire
    from gigapaxos_b200.spread import coordinator_of
    from helpers import Engine, group_descs_fast, make_config

    assert reps + 1 <= 8, "every round takes a slot of the window"
    members = [100, 101, 102]
    names = [f"NoopPaxosApp{i}" for i in range(G)]
    gids = np.array([g for g in range(G) if coordinator_of(names[g], members) == 100], np.uint32)
    engines = []
    for _ in range(2):
        e = Engine(lib, make_config(lib, max_groups=G, n_lanes=1, lane_node=[100], window=8, max_batch_recs=G,
                                    max_batch_payload=16 * G, log_ring_bytes=1 << 20))
        e.create_groups(group_descs_fast(G, members=tuple(members)))
        wire.set_group_names(e, gids, [names[g] for g in gids])
        engines.append(e)
    ed, eh = engines
    n = len(gids)

    def round_requests(r):
        return [wire.Request(names[g], 0, r * G + int(g), b"12345678", client=("10.0.0.1", 2000)) for g in gids]

    rounds = []
    for r in range(reps + 1):
        arena, refs = wire.pack_packets([wire.encode_request(q) for q in round_requests(r)])
        refs["node"] = 100
        rounds.append((torch.from_numpy(arena.copy()).pin_memory(),
                       torch.from_numpy(refs.view(np.uint8).reshape(n, 16).copy()).pin_memory(), round_requests(r)))
    d_arena = torch.empty(rounds[0][0].numel(), dtype=torch.uint8, device="cuda")
    d_refs = torch.empty((n, 16), dtype=torch.uint8, device="cuda")
    status = torch.empty(n, dtype=torch.int32, device="cuda")
    acc = torch.empty((n, 48), dtype=torch.uint8, device="cuda")
    heads = torch.empty(n, dtype=torch.int32, device="cuda")
    ctl = torch.zeros(8, dtype=torch.int32, device="cuda")
    h_out = torch.empty(256 * n, dtype=torch.uint8).pin_memory()
    h_refs = torch.empty((2 * n, 16), dtype=torch.uint8).pin_memory()
    caps = {"req": (n, 16 * n), "enc": (256 * n, 2 * n)}
    NOW = 1_700_000_000_000

    def device_leg(r):
        d_arena.copy_(rounds[r][0], non_blocking=True)
        d_refs.copy_(rounds[r][1], non_blocking=True)
        d = wire.decode_requests_device(ed, d_arena, d_refs, NOW, caps["req"])
        ctl.zero_()
        wire.propose_device_heads(ed, d.reqs, d.sizes[0], d.payload, d.sizes[1], status, acc, heads, ctl)
        enc = wire.encode_accepts_device(ed, acc, ctl.data_ptr(), d.sizes[0], heads, d.reqs, d.meta, d.sizes[0],
                                         d.payload, caps["enc"])
        caps["req"], caps["enc"] = d.sizes, enc.sizes
        h_out[: enc.sizes[0]].copy_(enc.out, non_blocking=True)
        h_refs[: enc.sizes[1]].copy_(enc.refs, non_blocking=True)
        torch.cuda.synchronize()
        return enc.sizes

    pay = np.zeros(16 * n, np.uint8)
    pay.reshape(n, 16)[:, :8] = np.frombuffer(b"12345678", np.uint8)
    host_reqs = np.zeros(n, abi.request_dtype)
    host_reqs["gid"], host_reqs["payload_off"], host_reqs["payload_len"] = gids, 16 * np.arange(n), 8
    host_reqs["entry_node"], host_reqs["client"] = 100, np.arange(n)
    host_out = {}

    def host_leg(r):
        reqs = host_reqs.copy()
        reqs["req_id"] = r * G + gids.astype(np.int64)
        a, _, st = eh.propose(reqs, pay)
        pk = []
        for x in a[np.argsort(a["gid"], kind="stable")]:  # the device encoder writes in gid order
            q = rounds[r][2][int(np.searchsorted(gids, x["gid"]))]
            q.entry_replica, q.entry_time = 100, NOW
            pk.append(wire.encode_accept(q, int(x["slot"]), int(x["bnum"]), int(x["bcoord"]), False,
                                         int(x["median_cp"]), int(x["sender"])))
        host_out[r] = pk
        return sum(len(b) for b in pk), len(pk)

    walls = {"device": [], "host": []}
    for r in range(reps + 1):  # round 0 warms both legs up
        for leg, run in (("device", device_leg), ("host", host_leg)):
            t = time.perf_counter()
            sizes = run(r)
            if r:
                walls[leg].append(time.perf_counter() - t)
            if leg == "device":
                dev_sizes = sizes
        # the same ACCEPT packets: each stored once, indexed for nodes 101 and 102
        refs = h_refs[: dev_sizes[1]].numpy().reshape(-1).view(abi.wire_ref_dtype)
        got = [bytes(h_out[int(f["off"]): int(f["off"]) + int(f["len"])].numpy()) for f in refs[::2]]
        assert got == host_out[r] and len(got) == n, "device and host ACCEPT packets differ"
    res = {"groups": G, "requests": n, "accept_bytes": int(dev_sizes[0]), "upload_bytes": int(rounds[0][0].numel() + 16 * n)}
    for leg in ("device", "host"):
        w = min(walls[leg])
        res[leg] = {"wall_s_min": w, "requests_per_s_wall": n / w}
    for e in engines:
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", choices=["coordinator_chain"], default=None,
                    help="run only this entry (at each --groups size)")
    args = ap.parse_args()
    import gigapaxos_b200
    from gigapaxos_b200 import abi, wire
    from helpers import Engine, group_descs_fast, make_config

    lib = gigapaxos_b200.load_library()
    res = {"card": card_info(), "runs": []}
    if args.only == "coordinator_chain":
        for G in args.groups:
            res["runs"].append({"groups": G, "coordinator_chain": coordinator_chain(lib, G, args.reps)})
        res["card_after"] = card_info()
        line = json.dumps(res)
        print(line)
        if args.out:
            with open(args.out, "w") as f:
                f.write(line + "\n")
        return
    tmp = tempfile.mkdtemp(prefix="gpx_wire_rate_")
    exe = os.path.join(tmp, "host_wire")
    src = os.path.join(tmp, "host_wire.c")
    open(src, "w").write(HOST_BENCH)
    subprocess.check_call(["gcc", "-O2", "-o", exe, src, "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "gigapaxos_b200", "libgpx.so"), "-lpthread",
                           "-Wl,-rpath," + os.path.join(ROOT, "gigapaxos_b200")])
    for G in args.groups:
        e = Engine(lib, make_config(lib, max_groups=G, n_lanes=1, lane_node=[101], window=8, max_batch_recs=G,
                                    max_batch_payload=1 << 20, log_ring_bytes=1 << 20))
        e.create_groups(group_descs_fast(G, members=(100, 101, 102)))
        names = [f"NoopPaxosApp{i}" for i in range(G)]
        gids = np.arange(G, dtype=np.uint32)
        wire.set_group_names(e, gids, names)
        # one ACCEPT per group (8-byte request value), as node 100 sends them to node 101
        t0 = time.time()
        pk = [wire.encode_accept(wire.Request(n, 0, i, b"12345678", entry_replica=100), 1, 0, 100, False, 0, 100)
              for i, n in enumerate(names)]
        arena, refs = wire.pack_packets(pk)
        gen_s = time.time() - t0
        status, acc, blob, _, _ = wire.decode_batch(e, pk)
        assert (status == abi.WS_OK).all() and len(acc) == G
        # replies in gpx_handle_accepts' layout, one per group, addressed to node 100; decisions one per group
        rep = np.zeros(G, abi.reply_dtype)
        rep["gid"], rep["slot"], rep["bnum"], rep["bcoord"], rep["who"] = gids, 1, 0, 100, abi.who(1, 0, 0)
        dec = np.zeros(G, abi.decision_dtype)
        dec["gid"], dec["slot"], dec["bnum"], dec["bcoord"], dec["flags"] = gids, 1, 0, 100, abi.F_DECISION
        calls = {"decode_accepts": lambda: wire.decode_batch(e, pk),
                 "encode_replies": lambda: wire.encode_replies(e, rep),
                 "encode_decisions": lambda: wire.encode_decisions(e, dec)}
        run = {"groups": G, "packet_gen_s": gen_s}
        for k, fn in calls.items():
            fn()  # warm-up
            walls = []
            for _ in range(args.reps):
                t = time.perf_counter()
                fn()  # ends in a device synchronise
                walls.append(time.perf_counter() - t)
            # the wall time includes the Python wrapper's own work; the bare C call is timed for decode below
            kms = [kernel_ms(fn) for _ in range(args.reps)]
            run[k] = {"packets": G, "wall_s_min": min(walls), "kernel_ms_min": min(kms),
                      "packets_per_s_kernels": G / (min(kms) / 1000.0), "packets_per_s_wall": G / min(walls)}
        # the bare C call (copies included, no Python record handling)
        import ctypes as C
        st = np.zeros(G, np.int32)
        a_out = np.zeros(G, abi.accept_dtype)
        b_out = np.zeros(len(blob) + 16, np.uint8)
        z = np.zeros(1, np.uint8)
        walls = []
        for _ in range(args.reps + 1):
            caps = [C.c_uint32(G), C.c_uint64(len(b_out)), C.c_uint32(0), C.c_uint32(0)]
            t = time.perf_counter()
            rc = lib.lib.gpx_wire_decode_batch(e.handle, C.c_uint32(G), abi._ptr(arena), C.c_uint64(len(arena)),
                                                abi._ptr(refs), abi._ptr(st), abi._ptr(a_out), C.byref(caps[0]),
                                                abi._ptr(b_out), C.byref(caps[1]), abi._ptr(z), C.byref(caps[2]),
                                                abi._ptr(z), C.byref(caps[3]))
            walls.append(time.perf_counter() - t)
            assert rc == 0
        run["decode_accepts"]["c_call_s_min"] = min(walls[1:])
        run["decode_accepts"]["packets_per_s_c_call"] = G / min(walls[1:])
        # host codec, one packet per call
        arena.tofile(os.path.join(tmp, "bytes"))
        refs.tofile(os.path.join(tmp, "refs"))
        T = os.cpu_count() or 1
        for mode, name in ((0, "host_decode_accept"), (1, "host_encode_batched_commit")):
            for threads in (1, T):
                s = min(float(subprocess.check_output([exe, os.path.join(tmp, "bytes"), os.path.join(tmp, "refs"),
                                                       str(mode), str(threads)]).decode())
                        for _ in range(args.reps))
                run[f"{name}_{threads}t"] = {"packets": G, "s_min": s, "packets_per_s": G / s, "threads": threads}
        e.close()
        run["acceptor_chain"] = acceptor_chain(lib, G, arena, refs, args.reps)
        run["coordinator_chain"] = coordinator_chain(lib, G, args.reps)
        res["runs"].append(run)
    res["card_after"] = card_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
