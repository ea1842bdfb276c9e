"""Project a submap collection into one mission-frame TSDF on the GPU (vgx_project_map) and mesh it, and
report where the time goes.

    python scripts/project_map.py [--workloads config2,config4] [--submaps N] [--repeats 5]
                                  [--min-weight 2.0] [--out FILE]

Input: bench.py's synthetic scenes (config2: 50 submaps at 0.2 m voxels; config4: 200 at 0.10 m), projected
at the scene's poses.  For each: the projection time (CUDA events around the call, and a host clock that
ends in a synchronise; the call includes the upload of the result: block hash, registration view, dense
grid), the kernel time of profiling slot 13 from a separate profiled call and its launch count, input and
output voxels, input voxels per second, the combined-mesh build time (vgx_mesh_build on the projected
map), and the device memory the first projection added (output submap plus the retained candidate and
sort scratch, from cudaMemGetInfo).  Two projections are checked bit-equal.  The card's name and power
limit are read in the same run.  Needs a GPU.
"""
import argparse

import _measure as M

OUT_ID = 0xFFFFFFF0


def measure(ctx, ids, T, min_weight, repeats):
    import torch
    from voxgraph_b200 import _lib
    n_in = 0
    for i in ids:
        _, vps, nb, _ = ctx.submap_info(i)
        n_in += nb * vps ** 3
    ctx.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    n_out_blocks = ctx.project_map(ids, T, OUT_ID)          # also the warm-up
    ctx.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    first = ctx.submap_download(OUT_ID)
    ctx.submap_free(OUT_ID)
    host, dev = [], []
    for _ in range(repeats):
        h, d, _ = M.timed(ctx, lambda: ctx.project_map(ids, T, OUT_ID))
        host.append(h)
        dev.append(d)
        ctx.submap_free(OUT_ID)
    kern_ms, launches, _ = M.profiled(ctx, _lib.VGX_SLOT_PROJECT, lambda: ctx.project_map(ids, T, OUT_ID))
    again = ctx.submap_download(OUT_ID)
    deterministic = all(a.tobytes() == b.tobytes() for a, b in zip(first, again))
    _, vps, _, _ = ctx.submap_info(OUT_ID)
    cfg = ctx.mesh_config(min_weight=min_weight)
    ctx.mesh_build([OUT_ID], None, cfg)                      # warm-up
    mesh_ms = [M.timed(ctx, lambda: ctx.mesh_build([OUT_ID], None, cfg))[0] for _ in range(repeats)]
    mesh_kern_ms, _, _ = M.profiled(ctx, _lib.VGX_SLOT_MESH, lambda: ctx.mesh_build([OUT_ID], None, cfg))
    xyz, tri = ctx.mesh_download()
    ctx.submap_free(OUT_ID)
    return dict(submaps=len(ids), input_voxels=n_in, output_blocks=n_out_blocks,
                output_voxels=n_out_blocks * vps ** 3,
                project_host_ms=[round(x, 3) for x in host], project_event_ms=[round(x, 3) for x in dev],
                project_best_ms=round(min(host), 3),
                input_voxels_per_s=float("%.4g" % (n_in / (min(host) / 1e3))),
                profiled_kernels_ms=round(kern_ms, 3), kernel_launches=launches,
                device_memory_added_bytes=int(free0 - free1), deterministic=deterministic,
                combined_mesh=dict(min_weight=min_weight, build_host_ms=[round(x, 3) for x in mesh_ms],
                                   build_best_ms=round(min(mesh_ms), 3), profiled_kernels_ms=round(mesh_kern_ms, 3),
                                   vertices=len(xyz), triangles=len(tri)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="config2,config4")
    ap.add_argument("--submaps", type=int, default=None)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--min-weight", type=float, default=2.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = dict(gpu=M.gpu_info(), results={})
    for name in a.workloads.split(","):
        w = M.WORKLOADS[name]
        ctx, sc, ids, T = M.upload_scene(w, a.submaps)
        r = measure(ctx, ids, T, a.min_weight, a.repeats)
        r["voxel_size"] = w["voxel_size"]
        res["results"][name] = r
        ctx.close()
        del sc
    M.emit(res, a.out)


if __name__ == "__main__":
    main()
