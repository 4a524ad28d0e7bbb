"""A pure-Python model of the response cache's key table (gpx_response_cache_*, include/gpx.h) and random cases for it.

The model restates the semantics of include/gpx.h, not the kernels: buckets of CELLS cells, the hash, put in input
order (same live key, else the lowest free or expired cell, else the oldest put time, lowest cell on a tie), expiry at
now_ms - put_ms >= timeout_ms, and match with the same-`client` rule and the name state's generations.
"""
from __future__ import annotations

import numpy as np

from helpers import abi

CELLS = 8
M64 = (1 << 64) - 1
GPX_EINVAL = abi.GPX_EINVAL

# RcCell of gigapaxos_b200/csrc/gpx_respcache.cuh: what the emulation's table holds
cell_dtype = np.dtype([("gid", "<u4"), ("gen", "<u4"), ("req_id", "<i8"), ("ip", "<u4"), ("port", "<u2"),
                       ("pad", "<u2"), ("handle", "<i4"), ("pad2", "<i4"), ("put_ms", "<i8")])
assert cell_dtype.itemsize == 40


def splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def ip_word(ip, port: int) -> int:
    """the client address as a big-endian word; an absent address (port 0) is 0 whatever its bytes"""
    if port == 0:
        return 0
    return (int(ip[0]) << 24) | (int(ip[1]) << 16) | (int(ip[2]) << 8) | int(ip[3])


def rc_hash(gid: int, gen: int, req_id: int, ip: int, port: int) -> int:
    """splitmix64(req_id ^ splitmix64(gid << 32 | gen) ^ splitmix64(ip << 16 | port))"""
    return splitmix64((req_id & M64) ^ splitmix64((gid << 32) | gen) ^ splitmix64((ip << 16) | port))


class Names:
    """the name state the cache reads: per gid its generation and whether it has a name; on = False is an engine
    without name state (generation 0, every gid counts as named)"""

    def __init__(self, G: int, on: bool = True):
        self.G, self.on = G, on
        self.gen = [0] * G
        self.named = [False] * G

    def name(self, gids):
        self.on = True
        for g in gids:
            self.gen[g] += 1
            self.named[g] = True

    def drop(self, gids):
        for g in gids:
            self.named[g] = False

    def gen_of(self, g: int) -> int:
        return self.gen[g] if self.on else 0

    def has_name(self, g: int) -> bool:
        return self.named[g] if self.on else True


class Cache:
    def __init__(self, n_buckets: int, timeout_ms: int, names: Names):
        self.nb, self.T, self.names = n_buckets, timeout_ms, names
        self.cells = [[None] * CELLS for _ in range(n_buckets)]  # (gid, gen, req_id, ip, port, handle, put_ms)

    def live(self, c, now: int) -> bool:
        return c is not None and (now < c[6] or now - c[6] < self.T)

    def _find(self, b, key, now):
        for i, c in enumerate(self.cells[b]):
            if self.live(c, now) and c[:5] == key:
                return i
        return -1

    def key_of(self, gid, req_id, ip, port):
        gen = self.names.gen_of(gid)
        k = (gid, gen, req_id, ip_word(ip, port), port)
        return k, rc_hash(*k) & (self.nb - 1)

    def put(self, keys: np.ndarray, now: int) -> int:
        """keys: abi rc_key_dtype records -> GPX_OK or GPX_EINVAL (nothing written)"""
        if any(int(k["handle"]) < 0 or int(k["gid"]) >= self.names.G for k in keys):
            return GPX_EINVAL
        for k in keys:
            key, b = self.key_of(int(k["gid"]), int(k["req_id"]), k["client_ip"], int(k["client_port"]))
            cells = self.cells[b]
            to = self._find(b, key, now)
            if to < 0:
                free = [i for i, c in enumerate(cells) if not self.live(c, now)]
                to = free[0] if free else min(range(CELLS), key=lambda i: (cells[i][6], i))
            cells[to] = key + (int(k["handle"]), now)
        return abi.GPX_OK

    def match(self, reqs: np.ndarray, meta: np.ndarray, now: int):
        """-> (hit int32 [n], indices of the misses in input order)"""
        clients = [int(c) for c in reqs["client"]]
        count = {}
        for c in clients:
            count[c] = count.get(c, 0) + 1
        hit = np.full(len(reqs), -1, np.int32)
        for q in range(len(reqs)):
            gid = int(reqs[q]["gid"])
            if count[clients[q]] > 1 or gid >= self.names.G or not self.names.has_name(gid):
                continue
            key, b = self.key_of(gid, int(reqs[q]["req_id"]), meta[q]["client_ip"], int(meta[q]["client_port"]))
            i = self._find(b, key, now)
            if i >= 0:
                hit[q] = self.cells[b][i][5]
        return hit, np.nonzero(hit < 0)[0]

    def table(self) -> np.ndarray:
        """the model's cells in the emulation's layout, [n_buckets * CELLS]; a free cell is all 0xff"""
        t = np.frombuffer(b"\xff" * (cell_dtype.itemsize * self.nb * CELLS), cell_dtype).copy()
        for b in range(self.nb):
            for i, c in enumerate(self.cells[b]):
                if c is not None:
                    r = t[b * CELLS + i]
                    r["gid"], r["gen"], r["req_id"], r["ip"], r["port"], r["handle"], r["put_ms"] = c
                    r["pad"], r["pad2"] = 0, 0
        return t


# ---- random cases ------------------------------------------------------------------------------------------------
IPS = [(10, 1, 2, 3), (10, 1, 2, 4), (192, 168, 0, 1)]
PORTS = [0, 4567, 4568]


def _addr(rng):
    port = int(rng.choice(PORTS))
    ip = IPS[int(rng.integers(len(IPS)))] if port or rng.integers(2) else (0, 0, 0, 0)
    return ip, port  # port 0 with a nonzero ip: the address is absent all the same


def random_keys(rng, n, G, pool):
    """n keys drawn from a small pool of (gid, req_id, address) so that keys collide on every field separately and
    repeat within one put"""
    k = np.zeros(n, abi.rc_key_dtype)
    for i in range(n):
        gid, req_id, (ip, port) = pool[int(rng.integers(len(pool)))]
        if rng.integers(4) == 0:  # one field changed
            f = int(rng.integers(4))
            gid = int(rng.integers(G)) if f == 0 else gid
            req_id = int(rng.choice([req_id + 1, -req_id - 1, (1 << 63) - 1, -(1 << 63)])) if f == 1 else req_id
            ip = IPS[int(rng.integers(len(IPS)))] if f == 2 else ip
            port = int(rng.choice(PORTS)) if f == 3 else port
        k[i]["gid"], k[i]["req_id"], k[i]["client_ip"], k[i]["client_port"] = gid, req_id, ip, port
        k[i]["handle"] = int(rng.integers(0, 1 << 31))
    return k


def random_requests(rng, n, G, pool, n_clients=None):
    """requests (abi.request_dtype) and their meta; some share a `client` value, as the requests of one batched
    RequestPacket do"""
    reqs = np.zeros(n, abi.request_dtype)
    meta = np.zeros(n, abi.req_meta_dtype)
    keys = random_keys(rng, n, G, pool)
    reqs["gid"], reqs["req_id"] = keys["gid"], keys["req_id"]
    meta["client_ip"], meta["client_port"] = keys["client_ip"], keys["client_port"]
    c, q = 0, 0
    while q < n:
        run = 1 if rng.integers(3) else int(rng.integers(2, 4))
        reqs["client"][q: q + run] = c
        c += 1 + int(rng.integers(0, 2))
        q += run
    perm = rng.permutation(n) if rng.integers(2) else np.arange(n)  # the same client need not be adjacent
    return reqs[perm], meta[perm]


def random_case(rng, G=8, n_ops=24):
    """-> (n_buckets, timeout_ms, names_on, ops): ops are ("put", keys, now), ("match", reqs, meta, now),
    ("name", gids) and ("drop", gids), with time steps that land exactly on the timeout"""
    n_buckets = int(rng.choice([1, 2, 4, 16]))
    T = int(rng.choice([0, 1, 50, 100]))
    names_on = bool(rng.integers(0, 4))
    pool = [(int(rng.integers(G)), int(rng.integers(-3, 1 << 40)), _addr(rng)) for _ in range(int(rng.integers(2, 9)))]
    now = int(rng.integers(0, 1000))
    ops = []
    if names_on:
        ops.append(("name", list(range(G))))
    for _ in range(n_ops):
        now += int(rng.choice([0, 1, T, max(T - 1, 0), T + 1, 7]))
        r = int(rng.integers(10))
        if r < 4:
            ops.append(("put", random_keys(rng, int(rng.integers(0, 40)), G, pool), now))
        elif r < 8:
            reqs, meta = random_requests(rng, int(rng.integers(1, 40)), G, pool)
            ops.append(("match", reqs, meta, now))
        elif names_on and r == 8:
            ops.append(("name", sorted(set(int(g) for g in rng.integers(0, G, size=3)))))
        elif names_on:
            ops.append(("drop", sorted(set(int(g) for g in rng.integers(0, G, size=2)))))
    return n_buckets, T, names_on, ops
