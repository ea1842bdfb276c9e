"""The pose-graph table layout (voxgraph_b200/csrc/graph_plan.cpp) on the host, without a GPU or the library:
the rank partition, the reduce tiles and their size, the off-diagonal block numbering, the items of every output
block, the per-block rank masks and the reduced offsets.  The tile cut fixes the order in which the constraint
sums add tile rows, and the multi-rank tables are what the peer exchange trusts, so every entry is checked here
for every rank of 1-8 ranks.  tests/cpp/graph_plan_test.cpp runs the plan of every rank for each case."""
import itertools
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "voxgraph_b200", "csrc")


def _define(name):
    text = open(os.path.join(CSRC, "graph_plan.h")).read()
    return int(re.search(r"#define %s (\d+)" % name, text).group(1))


SLOTS_PER_SM = _define("VGX_REG_TILE_SLOTS_PER_SM")
HW_UNITS = _define("VGX_REG_HW_TILE_UNITS")
UNIT = _define("VGX_REG_UNIT")
PACK_HDR = _define("PACK_HDR")


@pytest.fixture(scope="module")
def plan_exe(tmp_path_factory):
    from voxgraph_b200 import build
    nvcc = shutil.which(build._nvcc())
    assert nvcc, "nvcc not found: its include directory has int2 / int4"
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    exe = str(tmp_path_factory.mktemp("graph_plan") / "graph_plan_test")
    cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-I" + CSRC, "-I" + cuda_include,
           os.path.join(CSRC, "graph_plan.cpp"), os.path.join(ROOT, "tests", "cpp", "graph_plan_test.cpp"),
           "-o", exe]
    env = dict(os.environ)
    env.pop("CXX", None)
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    assert p.returncode == 0, p.stdout
    return exe


def case(N, cons, rel=(), nranks=1, constant=None, sms=132, override=0):
    """cons: (n, ref_node, read_node, grid_cells, grid16, locality_key) per constraint; rel: (a, b) per edge."""
    return dict(nranks=nranks, N=N, cons=[tuple(int(v) for v in c) for c in cons],
                rel=[tuple(int(v) for v in e) for e in rel], constant=[int(v) for v in (constant or [0] * N)], sms=sms,
                override=override)


def run(exe, cases):
    """-> [{"owner": [...], "plans": [plan of rank r, ...]}] per case."""
    lines = []
    for c in cases:
        lines.append("%d %d %d %d %d %d" % (c["nranks"], c["N"], len(c["cons"]), len(c["rel"]), c["sms"],
                                            c["override"]))
        lines.append(" ".join(map(str, c["constant"])))
        lines += [" ".join(map(str, k)) for k in c["cons"]]
        lines += ["%d %d" % e for e in c["rel"]]
    p = subprocess.run([exe], input="\n".join(lines) + "\n", stdout=subprocess.PIPE, text=True, check=True)
    out = [json.loads(line) for line in p.stdout.splitlines()]
    assert len(out) == len(cases)
    return out


def units(n):
    return (n + UNIT - 1) // UNIT


def tile_size(U, sms):
    slots = max(sms, 1) * SLOTS_PER_SM
    return min(HW_UNITS, max(4, -(-U // (2 * slots))))


def midpoint_owner(nranks, counts, keys):
    order = sorted(range(len(counts)), key=lambda i: keys[i])   # stable
    total = sum(max(n, 0) for n in counts)
    owner, before = [0] * len(counts), 0
    for i in order:
        n = max(counts[i], 0)
        r = ((2 * before + n) * nranks) // (2 * total) if total > 0 else 0
        owner[i] = min(max(r, 0), nranks - 1)
        before += n
    return owner


def check(c, out):
    """Every table of every rank against the layout rules, restated here."""
    N, cons, rel, nranks = c["N"], c["cons"], c["rel"], c["nranks"]
    owner = out["owner"]
    assert owner == midpoint_owner(nranks, [k[0] for k in cons], [k[5] for k in cons])
    # off-diagonal blocks: one per unordered node pair over all edges of all ranks, in first-appearance order
    block = {}
    for a, b in list(rel) + [(k[1], k[2]) for k in cons]:
        block.setdefault((min(a, b), max(a, b)), len(block))
    E = len(block)
    block_nodes = [v for pair in sorted(block, key=block.get) for v in pair]
    red, n_free = [], 0
    for i in range(N):
        red.append(-1 if c["constant"][i] else n_free)
        n_free += 0 if c["constant"][i] else 4
    mask = [0] * (N + E)
    for e, (a, b) in enumerate(rel):
        for ob in (a, b, N + block[(min(a, b), max(a, b))]):
            mask[ob] |= 1
    for i, (n, a, b, *_) in enumerate(cons):
        for ob in (a, b, N + block[(min(a, b), max(a, b))]):
            mask[ob] |= 1 << owner[i]
    seen = []
    for r, p in enumerate(out["plans"]):
        local = [i for i in range(len(cons)) if owner[i] == r]
        assert p["local"] == local
        seen += local
        assert p["residuals_local"] == sum(cons[i][0] for i in local)
        assert p["n_rel_local"] == (len(rel) if r == 0 else 0)
        # tiles: every local constraint cut in point order on unit boundaries, covered exactly once
        U = sum(units(cons[i][0]) for i in local)
        tu = c["override"] if c["override"] >= 1 else tile_size(U, c["sms"])
        assert p["tile_units"] == tu
        tiles, tb = p["tiles"], p["tile_begin"]
        assert len(tb) == len(local) + 1 and tb[0] == 0 and tb[-1] == len(tiles)
        unit0 = 0
        for k, i in enumerate(local):
            n, cells, grid16 = cons[i][0], cons[i][3], cons[i][4]
            mine = tiles[tb[k]:tb[k + 1]]
            assert [t[1] for t in mine] == list(range(0, n, tu * UNIT))
            for t in mine:
                assert t[0] == k and t[1] % UNIT == 0
                assert 0 < t[2] <= tu * UNIT and t[1] + t[2] <= n
                assert t[2] == min(tu * UNIT, n - t[1])
                assert t[3] == unit0
                unit0 += units(t[2])
                assert t[4] == (((cells + 7) & ~7) * 2 if grid16 and cells > 0 else 0)
            assert sum(t[2] for t in mine) == n
        assert p["n_units"] == unit0 == U
        assert p["grid_capacity"] == max([(cons[i][3] + 7) & ~7 for i in local if cons[i][4]], default=0)
        # blocks and items: local relative edges first (rank 0), then local constraints, with their roles
        assert p["E"] == E and p["block_nodes"] == block_nodes
        lists = [[] for _ in range(N + E)]
        srcs = [(-(e + 1), a, b) for e, (a, b) in enumerate(rel[:p["n_rel_local"]])]
        srcs += [(k, cons[i][1], cons[i][2]) for k, i in enumerate(local)]
        for s, a, b in srcs:
            t0, t1 = (tb[s], tb[s + 1]) if s >= 0 else (0, 0)
            lists[a].append([s, 0, t0, t1])
            lists[b].append([s, 1, t0, t1])
            lists[N + block[(min(a, b), max(a, b))]].append([s, 2 if a < b else 3, t0, t1])
        assert p["csr_begin"] == list(itertools.accumulate([len(li) for li in lists], initial=0))
        assert p["items"] == [it for li in lists for it in li]
        assert p["block_mask"] == mask
        csr = p["csr_begin"]
        for ob in range(N + E):   # bit r: exactly the blocks rank r has items for
            assert bool(mask[ob] >> r & 1) == (csr[ob + 1] > csr[ob]), (r, ob)
        assert p["red"] == red and p["n_free"] == n_free
        assert p["packed_len"] == PACK_HDR + 20 * N + 16 * E
    assert sorted(seen) == list(range(len(cons)))


def random_case(rs, nranks):
    N = int(rs.randint(2, 24))
    P = int(rs.randint(0, 40))
    cons = []
    for _ in range(P):
        a, b = rs.choice(N, 2, replace=False)
        n = 0 if rs.rand() < 0.1 else int(rs.randint(1, 6000))
        cons.append((n, a, b, rs.randint(0, 4097), rs.rand() < 0.7, rs.randint(0, 1000)))
    rel = [tuple(rs.choice(N, 2, replace=False)) for _ in range(int(rs.randint(0, N + 3)))]
    return case(N, cons, rel, nranks=nranks, constant=list(rs.rand(N) < 0.3),
                sms=int(rs.choice([1, 114, 132])), override=int(rs.choice([0, 0, 0, 1, 3, 129])))


@pytest.mark.parametrize("nranks", range(1, 9))
def test_every_rank_of_random_graphs(plan_exe, nranks):
    rs = np.random.RandomState(nranks)
    cases = [random_case(rs, nranks) for _ in range(30)]
    outs = run(plan_exe, cases)
    for c, out in zip(cases, outs):
        check(c, out)
    # some case spreads its constraints over every rank
    assert any(all(p["local"] for p in out["plans"]) for out in outs)


@pytest.mark.parametrize("sms", [114, 132])
def test_tile_size_at_its_edges(plan_exe, sms):
    e = 2 * sms * SLOTS_PER_SM
    expect = {3 * e: 4, 4 * e - 1: 4, 4 * e: 4, 4 * e + 1: 5, 63 * e: 63, 63 * e + 1: 64, 64 * e - 1: 64, 64 * e: 64,
              64 * e + 1: 64}
    cases = []
    for U in expect:
        # three constraints of U units in all, the last one ending inside a unit
        u = [U // 3, U // 3, U - 2 * (U // 3)]
        cases.append(case(4, [(u[0] * UNIT, 0, 1, 64, 1, 0), (u[1] * UNIT, 1, 2, 0, 0, 1),
                              (u[2] * UNIT - 5, 2, 3, 9, 1, 2)], sms=sms))
    for (U, tu), c, out in zip(expect.items(), cases, run(plan_exe, cases)):
        assert tile_size(U, sms) == tu and out["plans"][0]["tile_units"] == tu, U
        check(c, out)
    # the override replaces the rule whatever the size; values below 1 leave it in force
    overrides = [1, 3, 64, 129, 256, 0, -1]
    cases = [case(4, [(20000, 0, 1, 64, 1, 0), (31 * UNIT + 1, 1, 2, 0, 0, 1), (7, 2, 3, 9, 1, 2)], sms=sms,
                  override=o) for o in overrides]
    for o, c, out in zip(overrides, cases, run(plan_exe, cases)):
        assert out["plans"][0]["tile_units"] == (o if o >= 1 else 4)
        check(c, out)


def test_block_numbering_and_mirrored_pairs(plan_exe):
    # relative edges (0,1), (2,1); constraints (1,0), (0,1), (3,0), (0,3), (2,1): three blocks
    cons = [(100, 1, 0, 0, 0, 5), (40, 0, 1, 0, 0, 5), (33, 3, 0, 16, 1, 0), (0, 0, 3, 0, 0, 0), (64, 2, 1, 8, 1, 9)]
    c = case(4, cons, rel=[(0, 1), (2, 1)])
    out = run(plan_exe, [c])[0]
    check(c, out)
    p = out["plans"][0]
    assert p["E"] == 3 and p["block_nodes"] == [0, 1, 1, 2, 0, 3]
    assert p["tile_units"] == 4 and p["tile_begin"] == [0, 1, 2, 3, 3, 4]
    N = 4

    def items(ob):
        return p["items"][p["csr_begin"][ob]:p["csr_begin"][ob + 1]]
    # (source, role, tiles): role 2 when the block's rows are the item's first node, 3 when they are its second
    assert items(N + 0) == [[-1, 2, 0, 0], [0, 3, 0, 1], [1, 2, 1, 2]]
    assert items(N + 1) == [[-2, 3, 0, 0], [4, 3, 3, 4]]
    assert items(N + 2) == [[2, 3, 2, 3], [3, 2, 3, 3]]
    assert items(0) == [[-1, 0, 0, 0], [0, 1, 0, 1], [1, 0, 1, 2], [2, 1, 2, 3], [3, 0, 3, 3]]
    # on two ranks the numbering and the masks are the same, and only rank 0 evaluates the relative edges
    c2 = case(4, cons, rel=[(0, 1), (2, 1)], nranks=2)
    out2 = run(plan_exe, [c2])[0]
    check(c2, out2)
    p0, p1 = out2["plans"]
    assert p0["block_nodes"] == p1["block_nodes"] == p["block_nodes"] and p0["block_mask"] == p1["block_mask"]
    assert p1["n_rel_local"] == 0 and all(it[0] >= 0 for it in p1["items"])


def test_reduced_offsets_with_constant_nodes_anywhere(plan_exe):
    N = 6
    cons = [(50, 0, 5, 0, 0, 0), (70, 2, 3, 0, 0, 1)]
    cases = [case(N, cons, rel=[(0, 1), (1, 2), (3, 4)], constant=[m >> i & 1 for i in range(N)])
             for m in range(1 << N)]
    for c, out in zip(cases, run(plan_exe, cases)):
        check(c, out)
        p = out["plans"][0]
        free = [i for i in range(N) if not c["constant"][i]]
        assert p["n_free"] == 4 * len(free) and [p["red"][i] for i in free] == [4 * j for j in range(len(free))]


def test_edge_cases(plan_exe):
    cases = [case(1, []),                                   # one node, nothing else
             case(3, [], rel=[(0, 1), (1, 0), (2, 1)]),     # no registration constraints
             case(3, [(0, 0, 1, 0, 0, 0), (0, 1, 0, 5, 1, 3)], nranks=3),   # zero-point constraints only
             case(3, [(0, 0, 1, 0, 0, 0), (1, 1, 2, 0, 0, 1), (0, 2, 0, 0, 0, 2)], nranks=2)]
    outs = run(plan_exe, cases)
    for c, out in zip(cases, outs):
        check(c, out)
    p = outs[0]["plans"][0]
    assert p["E"] == 0 and p["tiles"] == [] and p["tile_begin"] == [0] and p["csr_begin"] == [0, 0]
    assert p["tile_units"] == 4 and p["n_units"] == 0 and p["grid_capacity"] == 0 and p["packed_len"] == PACK_HDR + 20
    p = outs[1]["plans"][0]
    assert p["E"] == 2 and p["tiles"] == [] and p["block_mask"] == [1] * 5
    zero = outs[2]
    assert zero["owner"] == [0, 0] and all(p["tiles"] == [] for p in zero["plans"])
    assert zero["plans"][0]["tile_begin"] == [0, 0, 0] and zero["plans"][1]["items"] == []
    assert [it[2:] for it in zero["plans"][0]["items"]] == [[0, 0]] * 6
