"""How even is the constraint -> rank partition in reduce-kernel TIME (not residual count)?
One GPU: for each rank r of an N-rank partition of the configs[3] workload, the registration constraints
the library would give to rank r are evaluated alone and their reduce kernel is timed.
  python scripts/shard_balance.py [nranks ...]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

sys.stdout = bench._REAL_STDOUT
w = dict(bench.WORKLOADS["config4"]); w["name"] = "config4"
sc = bench.build_scene(w)
from voxgraph_b200 import _lib, api  # noqa: E402

ctx = api.Context(0)
P = bench.Problem(ctx, api, sc)
reg = list(P.pg._registration)
cfgs = list(P.pg._reg_cfgs)
ref = np.array([r[0] for r in reg], np.uint32); read = np.array([r[1] for r in reg], np.uint32)
counts = np.array([ctx.submap_num_points(int(a), api.K_ISOSURFACE_POINTS) for a in ref], np.int32)


def kernel_us(sel):
    ctx.graph_set_registration_constraints_v(ref[sel], read[sel], [cfgs[i] for i in np.flatnonzero(sel)])
    for _ in range(4):
        ctx.graph_eval_async()
    ctx.synchronize()
    ctx.profile_reset(); ctx.profile_enable(True)
    for _ in range(6):
        ctx.graph_eval_async()
    ctx.synchronize()
    ms, n = ctx.profile_get(_lib.VGX_SLOT_REG_REDUCE)
    ctx.profile_enable(False)
    return ms / max(n, 1) * 1e3


full = kernel_us(np.ones(len(ref), bool))
print("all %d constraints on one GPU: reduce kernel %.1f us" % (len(ref), full))
for nr in [int(a) for a in sys.argv[1:]] or [2, 4, 8]:
    owner = api.shard_constraints(nr, counts, read)
    t = [kernel_us(owner == r) for r in range(nr)]
    res = [int(counts[owner == r].sum()) for r in range(nr)]
    print("N=%d  kernel us per rank: %s  max/mean %.3f  ideal %.1f  residuals per rank min/max %d/%d" % (
        nr, " ".join("%.1f" % v for v in t), max(t) / (sum(t) / nr), full / nr, min(res), max(res)))
ctx.close()
