"""What the timing scripts share: the card's description, bench.py's synthetic workloads uploaded to a
context, a timed call, a profiled call and the JSON result line.  Needs a GPU."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {"config2": dict(submaps=50, voxel_size=0.2, seed=2), "config4": dict(submaps=200, voxel_size=0.1, seed=4)}


def gpu_info():
    """The card's name, power limit and max SM clock, read by nvidia-smi in the run they describe."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:   # the figures are still reported, without the card's description
        return dict(error=str(e))


def upload_scene(workload, submaps=None):
    """bench.py's synthetic scene of workload (a WORKLOADS entry; submaps, when given, overrides its count),
    uploaded to a new context -> (ctx, scene, submap ids, T_M_S at the initial poses (n, 7) float32)."""
    from voxgraph_b200 import api, synth
    vs = workload["voxel_size"]
    sc = synth.make_scene(seed=workload["seed"], n_submaps=submaps or workload["submaps"], n_points=100,
                          voxel_size=vs, trunc=0.6 if abs(vs - 0.2) < 1e-9 else None, workers=os.cpu_count() or 1)
    ctx = api.Context(0)
    for s in sc.submaps:
        ctx.submap_upload(s.submap_id, s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)
    T = np.array([synth.pose_to_T(p) for p in sc.poses_init], np.float32)
    return ctx, sc, [s.submap_id for s in sc.submaps], T


def timed(ctx, fn):
    """fn() after a synchronise -> (host ms by a clock that ends in a synchronise, ms between CUDA events
    recorded around it on the context's stream, fn's result)."""
    import torch
    stream = torch.cuda.ExternalStream(ctx.stream_ptr)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ctx.synchronize()
    t = time.perf_counter()
    ev[0].record(stream)
    out = fn()
    ev[1].record(stream)
    ctx.synchronize()
    host = 1e3 * (time.perf_counter() - t)
    return host, ev[0].elapsed_time(ev[1]), out


def profiled(ctx, slot, fn):
    """fn() with kernel accounting on, from reset -> (kernel ms and launches of profiling slot `slot`, fn's
    result).  The other slots of the call stay readable through ctx.profile_get until the next reset."""
    ctx.profile_enable(True)
    ctx.profile_reset()
    out = fn()
    ms, launches = ctx.profile_get(slot)
    ctx.profile_enable(False)
    return ms, launches, out


def emit(result, out=None):
    """Print result as one JSON line, and append it to the file out when given."""
    line = json.dumps(result)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "a") as f:
            f.write(line + "\n")
