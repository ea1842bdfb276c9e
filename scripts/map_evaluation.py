"""Evaluate a projected submap map against a ground-truth TSDF on the GPU (vgx_map_evaluate, voxgraph's
MapEvaluation) and report where the time goes.

    python scripts/map_evaluation.py [--submaps 50] [--voxel-size 0.2] [--repeats 3] [--out FILE]

Input: bench.py's config 2 scene (50 submaps at 0.2 m voxels).  The ground truth covers the whole area: the
submaps projected at their true poses (sampled from the same synth world), then moved by a known offset, so the
alignment has a known answer.  The map is the submaps at their true poses.  Reported:
  - the stages, each bracketed by CUDA events on the context's stream and run through the same public entry
    points vgx_map_evaluate calls: projection, finish of the projected map (view, ESDF, relevant voxels), finish
    of the ground truth (view, ESDF), LM alignment, transform of the ground truth (+ its ESDF again), RMSE;
  - the whole vgx_map_evaluate call by a host clock ending in a synchronise (best of --repeats, each from a
    fresh copy of the ground truth);
  - the aligned pose against the known offset, the RMSE before and after;
  - the card's name, power limit and max SM clock, read in the same run.  Needs a GPU.
"""
import argparse

import numpy as np

import _measure as M

GT_ID = 0xFFFFFF00
PROJ_ID = 0xFFFFFF01
OFFSET = (0.1, -0.05, 0.03, 0.01)   # where the ground truth is moved to: the alignment should undo it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--submaps", type=int, default=50)
    ap.add_argument("--voxel-size", type=float, default=0.2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from voxgraph_b200 import api, synth
    ctx, sc, ids, _ = M.upload_scene(dict(submaps=a.submaps, voxel_size=a.voxel_size, seed=2))
    vps = sc.submaps[0].vps
    T = np.array([synth.pose_to_T(p) for p in sc.poses_gt], np.float32)
    # the ground truth: the whole area at the true poses, moved by the inverse of OFFSET (so that the alignment
    # should find OFFSET)
    ctx.project_map(ids, T, GT_ID)
    x, y, z, yaw = OFFSET   # T(OFFSET).inverse() = (yaw -yaw, translation -R(-yaw) t)
    c, s_ = np.cos(-yaw), np.sin(-yaw)
    Tinv = synth.pose_to_T([-(c * x - s_ * y), -(s_ * x + c * y), -z, -yaw])
    ctx.submap_transform(GT_ID, Tinv)
    gt_layer = ctx.submap_download(GT_ID)
    gt_vs = ctx.submap_info(GT_ID)[0]

    def fresh_gt():
        ctx.submap_upload(GT_ID, gt_vs, vps, *gt_layer)

    # the stages, through the public entry points
    fresh_gt()
    filt = ctx.registration_filter(min_voxel_weight=1.0, max_voxel_distance=0.3, use_esdf_distance=1)
    stages = {}
    _, stages["projection_ms"], _ = M.timed(ctx, lambda: ctx.project_map(ids, T, PROJ_ID))

    def finish_projected():
        ctx.submap_finish(PROJ_ID)
        ctx.submap_generate_esdf(PROJ_ID)
        ctx.submap_extract_points(PROJ_ID, filt)

    def finish_gt():
        ctx.submap_finish(GT_ID)
        ctx.submap_generate_esdf(GT_ID)

    _, stages["finish_projected_ms"], _ = M.timed(ctx, finish_projected)
    _, stages["finish_ground_truth_ms"], _ = M.timed(ctx, finish_gt)
    before = ctx.evaluate_layers_rmse(GT_ID, PROJ_ID)
    ctx.graph_set_nodes([PROJ_ID, GT_ID], np.zeros((2, 4)), np.array([1, 0], np.uint8))
    ctx.graph_set_registration_constraints([PROJ_ID], [GT_ID], ctx.reg_config(
        registration_point_type=api.K_VOXELS, no_correspondence_cost=0.0, sampling_ratio=-1.0,
        use_esdf_distance=1))
    opts = ctx.solver_options(max_num_iterations=200, parameter_tolerance=1e-12, max_solver_time_s=1e9)
    _, stages["lm_ms"], (x, summ) = M.timed(ctx, lambda: ctx.graph_solve(2, opts))
    pose = x[1]
    Tal = synth.pose_to_T(pose)

    def transform():
        ctx.submap_transform(GT_ID, Tal)
        finish_gt()

    _, stages["transform_ms"], _ = M.timed(ctx, transform)
    _, stages["rmse_ms"], after = M.timed(ctx, lambda: ctx.evaluate_layers_rmse(GT_ID, PROJ_ID))
    ctx.graph_set_nodes([], np.zeros((0, 4)), np.zeros(0, np.uint8))
    ctx.submap_free(PROJ_ID)
    # the whole call
    host = []
    for _ in range(a.repeats):
        fresh_gt()
        h, _, r = M.timed(ctx, lambda: ctx.map_evaluate(GT_ID, ids, T))
        host.append(h)
    res = dict(gpu=M.gpu_info(), submaps=len(ids), voxel_size=a.voxel_size,
               ground_truth_blocks=int(len(gt_layer[0])),
               stages_event_ms={k: round(v, 3) for k, v in stages.items()},
               map_evaluate_host_ms=[round(h, 3) for h in host], map_evaluate_best_ms=round(min(host), 3),
               offset=list(OFFSET), aligned_pose=[float(v) for v in r.aligned_pose],
               stage_aligned_pose=[float(v) for v in pose], lm_iterations=int(r.summary.iterations),
               termination=int(r.summary.termination),
               rmse_before=float(before.rmse), rmse_after=float(r.details.rmse),
               evaluated_voxels=int(r.details.num_evaluated_voxels))
    ctx.close()
    M.emit(res, a.out)


if __name__ == "__main__":
    main()
