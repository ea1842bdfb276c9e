"""Save and load a submap collection file (cblox SubmapCollection stream) on the GPU and report where
the time goes.

    python scripts/collection_io.py --workload config2 [--submaps N] [--repeats 3] [--out FILE]

The scene is bench.py's synthetic one (config2: 50 submaps at 0.2 m voxels; config4: 200 submaps at
0.10 m; --submaps shrinks it).  Reported per direction, from un-profiled calls: wall time, GB/s of file
and voxels/s; from separate profiled calls (CUDA events around each phase, so they are slower): the split
into the codec kernels, the host <-> device stream copies and, for a load, the upload (block hash,
registration view, grid).  Host framing is timed on its own through vgx_collection_scan, which runs the
same parser as a load.  The card's name and power limit are read in the same run.  Needs a GPU.
"""
import argparse
import time

import _measure as M


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="config2", choices=sorted(M.WORKLOADS))
    ap.add_argument("--submaps", type=int, default=None)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from voxgraph_b200 import _lib, api
    w = M.WORKLOADS[a.workload]
    t0 = time.time()
    ctx, sc, ids, T = M.upload_scene(w, a.submaps)
    t_scene = time.time() - t0
    n_blocks = sum(s.num_blocks for s in sc.submaps)
    n_vox = n_blocks * sc.submaps[0].vps ** 3
    observed = int(sum((s.weight > 1e-6).sum() for s in sc.submaps))

    data = ctx.collection_save(ids, T)   # warm-up: staging buffers, module load
    ctx2 = api.Context(0)

    def save():
        host, _, out = M.timed(ctx, lambda: ctx.collection_save(ids, T))
        assert out == data
        return host

    def free_loaded():
        for i in ids:
            try:
                ctx2.submap_free(i)
            except api.VgxError:
                pass

    def load():
        free_loaded()
        return M.timed(ctx2, lambda: ctx2.collection_load(data))[0]

    def split(c, fn):
        """fn's codec kernel, stream copy and upload time from one profiled call."""
        codec_ms, _, _ = M.profiled(c, _lib.VGX_SLOT_COLL_CODEC, fn)
        return dict(codec_kernels_ms=round(codec_ms, 3),
                    stream_copies_ms=round(c.profile_get(_lib.VGX_SLOT_COLL_COPY)[0], 3),
                    upload_ms=round(c.profile_get(_lib.VGX_SLOT_COLL_UPLOAD)[0], 3))

    load()
    save_t = [save() for _ in range(a.repeats)]
    load_t = [load() for _ in range(a.repeats)]
    save_split = split(ctx, lambda: ctx.collection_save(ids, T))
    free_loaded()
    load_split = split(ctx2, lambda: ctx2.collection_load(data))
    scan_t = []
    for _ in range(a.repeats):
        t = time.perf_counter()
        api.Context.collection_scan(data)
        scan_t.append(time.perf_counter() - t)
    # the loaded map is the saved one
    for s in sc.submaps[:3]:
        assert ctx2.submap_download(s.submap_id)[1].tobytes() == ctx.submap_download(s.submap_id)[1].tobytes()

    def rates(ts):
        best = min(ts)
        return dict(wall_ms=[round(x, 3) for x in ts], best_ms=round(best, 3),
                    file_GBps=round(len(data) / best / 1e6, 3), voxels_per_s=float("%.4g" % (n_vox / best * 1e3)))

    M.emit(dict(
        workload=a.workload, submaps=len(ids), blocks=n_blocks, voxels=n_vox, observed_voxels=observed,
        voxel_size=w["voxel_size"], file_bytes=len(data), file_bytes_per_voxel=round(len(data) / n_vox, 3),
        hbm_bytes_per_voxel=8, scene_build_s=round(t_scene, 1), gpu=M.gpu_info(),
        save=dict(rates(save_t), profiled_split_ms=save_split),
        load=dict(rates(load_t), host_framing_ms=round(1e3 * min(scan_t), 3), profiled_split_ms=load_split)), a.out)
    ctx.close()
    ctx2.close()


if __name__ == "__main__":
    main()
