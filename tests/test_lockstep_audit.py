"""Which kernels read or write the group-state planes that a VALID lockstep record leaves stale, and how each of them
is kept off stale words (CPU; reads the sources only).

k_round_g<L, true> keeps a group whose lanes advance in lockstep as one record (gpx_dev.cuh, ls_rec) and leaves that
group's acc_row, coord_row[cl] and ns_u[cl] words (and node_slots[cl], which ns_u says is stale) behind.  A kernel that
reads those words must run after ls_settle, or read only words a VALID record keeps current.  Nothing crashes when a
settle is missing: the kernel answers from a slot one or more rounds old.  So every kernel whose body, or any device
function or macro it reaches, names a plane word is listed below with the reason it never sees a stale one, and a new
such kernel, or a new launch of a listed one, fails this test until the table says how it is settled.

For kernels that are settled, the test also checks each host function that launches them: an ls_settle call comes
before the launch in that function, or the function is one of the launch helpers that settle (gpx_engine.cu).
"""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gigapaxos_b200", "csrc")

PLANE_WORDS = {"acc_row", "coord_row", "ns_u", "node_slots"}

SETTLED, CURRENT, OWNER = "settled", "current", "owner"
# kernel -> (reason, {host function that launches it: how the launch is settled}).  "settles": ls_settle comes
# earlier in the same function; "<helper>": the launch is in a helper that settles first, or whose only callers do.
PLANE_KERNELS = {
    "k_propose": (SETTLED, {"launch_propose": "settles"}),
    "k_accept": (SETTLED, {"launch_accept": "settles"}),
    "k_act": (SETTLED, {"launch_accept": "settles"}),
    "k_tally": (SETTLED, {"launch_tally": "settles"}),
    "k_tally_slots": (SETTLED, {"launch_tally": "settles"}),
    "k_commit": (SETTLED, {"launch_commit": "settles"}),
    "k_init_groups": (SETTLED, {"gpx_create_groups": "settles"}),
    "k_destroy_groups": (SETTLED, {"gpx_destroy_groups": "settles"}),
    "k_dump_rows": (SETTLED, {"gpx_dump_rows": "settles"}),
    "k_load_rows": (SETTLED, {"gpx_load_rows": "settles"}),
    "k_patch": (SETTLED, {"gpx_patch": "settles"}),
    "k_get_flags": (SETTLED, {"gpx_get_group_flags": "settles"}),
    "k_select_groups": (SETTLED, {"gpx_select_groups": "settles"}),
    "k_missing_decisions": (SETTLED, {"gpx_missing_decisions": "settles"}),
    "k_pause_groups": (SETTLED, {"gpx_pause_groups": "settles"}),
    "k_prepare": (SETTLED, {"gpx_handle_prepares": "settles"}),
    "k_prepare_tally": (SETTLED, {"gpx_handle_prepare_replies": "settles"}),
    "k_sp_tally": (SETTLED, {"spread_enqueue": "gpx_spread_round"}),
    "k_sp_commit": (SETTLED, {"spread_enqueue": "gpx_spread_round"}),
    "k_sp_accept": (SETTLED, {"spread_enqueue": "gpx_spread_round"}),
    # the team kernel and k_round_g<L, false> run after launch_round settled (round_uses_ls is false for them);
    # k_round_g<L, true> owns the records, and k_round_slow only takes groups whose record k_round_g wrote back first
    "k_round": (OWNER, {"launch_round_t": "launch_round"}),
    "k_round_g": (OWNER, {"launch_round_t": "launch_round"}),
    "k_round_slow": (OWNER, {"launch_round_t": "launch_round"}),
    "k_ls_settle": (OWNER, {"ls_settle": "the settle itself"}),
    # request routing (propose_route) reads the entry lane's and the ballot coordinator's acc_row ballot and coord_row
    # ballot and EXISTS bit: a VALID record never changes a ballot or EXISTS (gpx_dev.cuh), so those words are current
    "k_wire_fwd": (CURRENT, {}),
    "k_json_enc_fwd": (CURRENT, {}),
}


def strip(src):
    """comments and string / character literals blanked, line structure kept"""
    src = re.sub(r"/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    return re.sub(r"\"(\\.|[^\"\\\n])*\"|'(\\.|[^'\\\n])*'", '""', src)


def macros(src):
    """#define NAME ... (with continuation lines) -> {NAME: body}; the source with every preprocessor line blanked"""
    out, lines, keep = {}, src.split("\n"), []
    i = 0
    while i < len(lines):
        line = lines[i]
        if line.lstrip().startswith("#"):
            block = [line]
            while block[-1].endswith("\\") and i + 1 < len(lines):
                i += 1
                block.append(lines[i])
            m = re.match(r"\s*#\s*define\s+(\w+)(.*)", " ".join(b.rstrip("\\") for b in block), flags=re.S)
            if m:
                out.setdefault(m.group(1), "")
                out[m.group(1)] += " " + m.group(2)
            keep.extend([""] * len(block))
        else:
            keep.append(line)
        i += 1
    return out, "\n".join(keep)


def functions(src):
    """[(name, is_kernel, body)] of every function defined at namespace or struct level (struct, namespace and
    extern blocks are transparent)"""
    out, i, n = [], 0, len(src)
    start = 0  # where the current declaration began
    while i < n:
        c = src[i]
        if c in ";}":
            start = i + 1
        elif c == "{":
            head = src[start:i]
            flat = re.sub(r"__launch_bounds__\s*\([^)]*\)|__align__\s*\([^)]*\)", " ", head)
            m = re.search(r"(~?\w+)\s*\(", flat)
            if re.match(r"\s*(template\s*<[^>]*>\s*)?(struct|class|union|enum|namespace)\b|\s*extern\b", flat) or not m \
                    or m.group(1) in ("if", "for", "while", "switch", "sizeof", "static_assert") or "=" in flat[: m.start()]:
                start = i + 1  # a transparent block (or an initializer, which holds no function)
            else:
                d, j = 0, i
                while j < n:
                    if src[j] == "{":
                        d += 1
                    elif src[j] == "}":
                        d -= 1
                        if d == 0:
                            break
                    j += 1
                out.append((m.group(1), "__global__" in head, src[i: j + 1]))
                i, start = j, j + 1
        i += 1
    return out


def ids(text):
    return set(re.findall(r"\b[A-Za-z_]\w*\b", text))


def device_sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))


def device_bodies():
    """({device function or macro: the identifiers of its body}, {kernel names})"""
    bodies, kernels = {}, set()
    for f in device_sources():
        ms, src = macros(strip(open(os.path.join(CSRC, f)).read()))
        for name, body in ms.items():
            bodies[name] = bodies.get(name, set()) | ids(body)
        for name, is_kernel, body in functions(src):
            bodies[name] = bodies.get(name, set()) | ids(body)
            if is_kernel:
                kernels.add(name)
    return bodies, kernels


def reach(bodies, name, skip=frozenset()):
    """the plane words `name` names, directly or through the functions and macros it calls (other than `skip`)"""
    seen, todo, w = set(), [name], set()
    while todo:
        f = todo.pop()
        if f in seen or f in skip:
            continue
        seen.add(f)
        b = bodies.get(f, set())
        w |= b & PLANE_WORDS
        todo.extend(b & bodies.keys())
    return w


def plane_kernels():
    """{kernel: the plane words it reaches, directly or through device functions and macros}"""
    bodies, kernels = device_bodies()
    out = {k: reach(bodies, k) for k in kernels}
    return {k: w for k, w in out.items() if w}


def host_functions():
    """{host function: body} of gpx_engine.cu and the host files it includes"""
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".inc", ".cpp")):
            _, src = macros(strip(open(os.path.join(CSRC, f)).read()))
            for name, _, body in functions(src):
                out[name] = out.get(name, "") + body
    return out


def launch_sites(host, kernel):
    return {name for name, body in host.items() if re.search(rf"\b{kernel}\b", body)}


def test_the_scan_sees_every_kernel_and_its_helpers():
    found = plane_kernels()
    # a direct reference, one through a device function, one through a helper two calls deep
    assert found["k_load_rows"] >= {"acc_row", "coord_row", "node_slots"}
    assert "acc_row" in found["k_dump_rows"] and "acc_row" in found["k_wire_fwd"]
    assert "k_md5" not in found and "k_log_scan" not in found


def test_every_kernel_that_reaches_the_planes_says_how_it_is_settled():
    found = set(plane_kernels())
    assert not found - PLANE_KERNELS.keys(), (
        f"kernels that read or write acc_row / coord_row / ns_u / node_slots with no entry in PLANE_KERNELS: "
        f"{sorted(found - PLANE_KERNELS.keys())}; settle before launching them (ls_settle, gpx_engine.cu) and say so")
    assert not PLANE_KERNELS.keys() - found, f"stale entries: {sorted(PLANE_KERNELS.keys() - found)}"


@pytest.mark.parametrize("kernel", sorted(k for k, (why, _) in PLANE_KERNELS.items() if why != CURRENT))
def test_every_launch_of_a_plane_kernel_is_settled(kernel):
    host = host_functions()
    sites = launch_sites(host, kernel)
    why, table = PLANE_KERNELS[kernel]
    assert sites == set(table), f"{kernel} is launched from {sorted(sites)}, the table names {sorted(table)}"
    for fn, how in table.items():
        body = host[fn]
        at = re.search(rf"\b{kernel}\b", body).start()
        if how == "settles":
            # textual order only: a settle on one branch and the launch on another would pass.  Every settling
            # function today settles unconditionally right before its launch; the GPU tests catch the rest.
            s = body.find("ls_settle(")
            assert 0 <= s < at, f"{fn} launches {kernel} without an ls_settle before it"
        elif how == "launch_round":
            lr = host["launch_round"]
            assert re.search(r"if \(round_uses_ls\(e\)\)\s*e->ls_live = true;\s*else\s*ls_settle\(e, st\);", lr), \
                "launch_round settles unless k_round_g<L, true> takes the round"
            assert lr.find("ls_settle(") < lr.find("launch_round_t<")
            assert launch_sites(host, "launch_round_t") == {"launch_round"}
        elif how == "gpx_spread_round":
            sr = host["gpx_spread_round"]
            assert 0 <= sr.find("ls_settle(") < sr.find(f"{fn}("), f"gpx_spread_round settles before {fn}"
            assert launch_sites(host, fn) == {"gpx_spread_round"}
        else:
            assert kernel == "k_ls_settle"


def test_every_call_of_a_launch_helper_is_after_its_settle():
    """the launch helpers settle first thing, so a new caller of theirs needs no settle of its own"""
    host = host_functions()
    for helper in ("launch_propose", "launch_accept", "launch_tally", "launch_commit"):
        body = host[helper]
        first_launch = min(m.start() for m in re.finditer(r"\bk_\w+\b|GPX_DISPATCH_L", body))
        assert 0 <= body.find("ls_settle(e, st);") < first_launch, helper


def test_the_forwards_encoders_read_only_ballots_and_exists():
    """k_wire_fwd and k_json_enc_fwd do not settle: they route through propose_route, which reads the ballot of
    acc_row (.y, .z) and the ballot and EXISTS bit of coord_row (.x, .y, .w).  A VALID record keeps all of those
    current; a change to propose_route that reads another plane field (a slot, the GC slot, a node slot) fails here"""
    src = strip(open(os.path.join(CSRC, "gpx_dev.cuh")).read())
    body = next(b for name, _, b in functions(macros(src)[1]) if name == "propose_route")
    for var in re.findall(r"const int4 (\w+) = S\.(?:acc_row|coord_row)\[", body):
        used = set(re.findall(rf"\b{var}\.(\w)", body))
        allowed = {"y", "z"} if var.startswith("A") else {"x", "y", "w"}
        assert used <= allowed, (var, used)
    assert not ids(body) & {"ns_u", "node_slots", "ls_rec", "ns_get", "ns_load"}
    # and propose_route is the encoders' only way to the planes: nothing else they call, nor their own bodies, names
    # a plane word
    bodies, _ = device_bodies()
    for k in ("k_wire_fwd", "k_json_enc_fwd"):
        assert reach(bodies, k) <= {"acc_row", "coord_row"}
        assert not reach(bodies, k, skip=frozenset({"propose_route"})), f"{k} reaches the planes past propose_route"
