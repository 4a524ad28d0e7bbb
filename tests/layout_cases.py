"""Named engine layouts for the layout-aware fuzzer (tests/fuzz.py): the node each lane serves and the member lists of
the groups (gid g gets members[g % len(members)]).  Each one is there to reach code that the default layout -- lane l
serves member l of every group -- never does.  Nodes 900 and up are served by no lane: remote members."""
from __future__ import annotations

from itertools import combinations

import numpy as np
import pytest

from helpers import Engine, GpxErrorT, abi, group_descs, make_config

N8 = [100, 101, 102, 103, 104, 105, 106, 107]
REM = list(range(900, 916))

LAYOUTS = {
    # identity groups, R = L: k_round's team kernel with 32 mod L idle lanes per warp (L = 5, 6, 7), median_regs with an
    # even count (4, 6, 8), every lane count the phase kernels are instantiated for beyond the default 3
    "ident4": dict(lane_node=N8[:4], members=[N8[:4]]),
    "ident5": dict(lane_node=N8[:5], members=[N8[:5]]),
    "ident6": dict(lane_node=N8[:6], members=[N8[:6]]),
    "ident7": dict(lane_node=N8[:7], members=[N8[:7]]),
    "ident8": dict(lane_node=N8[:8], members=[N8[:8]]),
    # every member local, lane order != member order: round_general's dstIdx / lane_of_idx mapping
    "perm3": dict(lane_node=[102, 100, 101], members=[[101, 100, 102]]),
    # the same at 5 lanes, with the members of one group listed in yet another order
    "perm5": dict(lane_node=[103, 100, 104, 102, 101], members=[[104, 103, 102, 101, 100], [100, 101, 102, 103, 104]]),
    # every 3-member subset of 5 lanes: ten member sets, two lanes outside each group (dst_mask = lane_mask, rows of
    # non-member lanes)
    "sub3of5": dict(lane_node=N8[:5], members=[list(c) for c in combinations(N8[:5], 3)]),
    # every 5- and 3-member subset of 8 lanes: 112 member sets, propose_route to a coordinator lane other than the
    # entry lane, tally_reply instead of the identity fast path
    "sub5of8": dict(lane_node=N8, members=[list(c) for c in combinations(N8, 5)] + [list(c) for c in combinations(N8, 3)]),
    # local and remote members, 1 to 16 of them, lanes in no order: remote coordinators (GPX_RS_FORWARD), groups whose
    # local members are a minority, median_minus with 9-16 members
    "remote": dict(lane_node=[104, 100, 102, 101], members=[
        [100], [100, 900], [101, 900, 901], [100, 101, 102, 900], [102, 900, 901, 902, 903],
        [100, 101, 102, 104, 900, 901, 902, 903, 904], [101, 102] + REM[:10], [100, 101, 102, 104] + REM[:12],
        [104] + REM[:15]]),
    # all 8 lanes and 8 remote members in one group of 16, with 8- and 12-member groups beside it
    "remote8": dict(lane_node=N8[::-1], members=[N8 + REM[:8], N8[2:6] + REM[:8], N8[:6] + REM[:2], N8]),
    # group sizes 1 to 6 in one 6-lane engine, identity groups among them
    "mixed": dict(lane_node=N8[:6], members=[[100], [100, 101], [102, 103, 104], N8[:6], [101, 103, 105, 900],
                                             [104, 105], N8[:4], N8[1:6]]),
}

# layouts with a remote member in some group
REMOTE_LAYOUTS = {k for k, v in LAYOUTS.items() if any(m >= REM[0] for ms in v["members"] for m in ms)}
# layouts with a group of more than GPX_MAX_LANES members
BIG_LAYOUTS = {k for k, v in LAYOUTS.items() if any(len(ms) > 8 for ms in v["members"])}


def is_ident(f, g: int) -> bool:
    """the engine's GPX_META_IDENT: the sorted members are exactly the lanes, lane l serving member l"""
    return f.members[g] == f.lane_node


def decided_gids(f) -> set:
    """the groups some lane executed at least one slot of"""
    return {g for h in f.history for g, seq in h.items() if seq}


def assert_reached(f, name):
    """the layout reached what it is there for: decisions in groups that are not GPX_META_IDENT, requests forwarded
    to a remote coordinator, decisions in groups of more than 8 members"""
    dg = decided_gids(f)
    assert len(dg) > f.G // 4, f"{name}: only {len(dg)} groups decided"
    if not name.startswith("ident"):
        assert any(not is_ident(f, g) for g in dg), name
    if name in REMOTE_LAYOUTS:
        assert f.n_forward > 0, name
    if name in BIG_LAYOUTS:
        assert any(len(f.members[g]) > 8 for g in dg), name


# ---- input rules shared by the engine and the oracle ---------------------------------------------------------------
MAX_MSETS = 4096  # GPX_MAX_MSETS (include/gpx.h)


def descs(members_list, gid0=0):
    """one group desc per member list (as listed, unsorted), gids gid0.."""
    d = group_descs(len(members_list), members=(), gid0=gid0)
    for k, m in enumerate(members_list):
        d["n_members"][k] = len(m)
        d["members"][k, :len(m)] = m
    return d


def small_engine(lib, **kw):
    cfg = dict(max_groups=64, n_lanes=3, lane_node=[100, 101, 102], max_group_size=4, max_batch_recs=1 << 13,
               max_batch_payload=1 << 18)
    cfg.update(kw)
    return Engine(lib, make_config(lib, **cfg))


def refused(code, fn, *a, **kw):
    with pytest.raises(GpxErrorT) as ex:
        fn(*a, **kw)
    assert ex.value.code == code, ex.value


def all_rows(e, G):
    return [e.dump_rows(np.arange(G), lane).tobytes() for lane in range(e.n_lanes)]


def check_input_rules(lib):
    """two lanes may not serve one node, a group lists a node once and has at most max_group_size members, gids and
    lanes are in range: the call is refused (GPX_EINVAL at creation, GPX_ERANGE for groups and rows) and changes
    nothing, whichever of its records breaks the rule"""
    refused(abi.GPX_EINVAL, small_engine, lib, lane_node=[100, 101, 100])
    refused(abi.GPX_EINVAL, small_engine, lib, max_group_size=17)
    e = small_engine(lib)
    e.create_groups(descs([[100, 101, 102]] * 4))
    before = all_rows(e, 64)
    refused(abi.GPX_ERANGE, e.create_groups, descs([[100, 101, 103], [100, 101, 101]], gid0=4))
    refused(abi.GPX_ERANGE, e.create_groups, descs([[100, 101, 104], [100, 101, 102, 103, 104]], gid0=4))
    refused(abi.GPX_ERANGE, e.create_groups, np.concatenate([descs([[100, 101, 105]], gid0=4), descs([[100]], gid0=64)]))
    assert all_rows(e, 64) == before
    rows = e.dump_rows(np.arange(4), 0)
    dup = rows.copy()
    dup["members"][1, 1] = dup["members"][1, 0]
    refused(abi.GPX_ERANGE, e.load_rows, dup)
    big = rows.copy()
    big["n_members"][2] = 5
    big["members"][2, 3:5] = [103, 104]
    refused(abi.GPX_ERANGE, e.load_rows, big)
    lane = rows.copy()
    lane["lane"][3] = 3
    refused(abi.GPX_ERANGE, e.load_rows, lane)
    assert all_rows(e, 64) == before
    e.close()


def mset_limit_engine(lib):
    """an engine whose member-set table is full: MAX_MSETS - 1 distinct sets, a call that would add two more is refused
    whole, one more goes, the next new one is refused, a known set listed in another order still goes.  Groups
    0 .. MAX_MSETS + 1 are live."""
    e = small_engine(lib, max_groups=MAX_MSETS + 8)
    e.create_groups(descs([[100, 101, 1000 + k] for k in range(MAX_MSETS - 1)]))
    refused(abi.GPX_ERANGE, e.create_groups, descs([[100, 101, 999], [100, 102, 5000]], gid0=MAX_MSETS - 1))
    e.create_groups(descs([[100, 101, 999]], gid0=MAX_MSETS - 1))
    refused(abi.GPX_ERANGE, e.create_groups, descs([[100, 102, 5000]], gid0=MAX_MSETS))
    e.create_groups(descs([[1000, 101, 100], [101, 1001, 100]], gid0=MAX_MSETS))
    return e
