"""CPU checks of the map-evaluation rules: the RMSE restatement (tests/rmse_exact.py) against hand-derived
answers for every branch, the transform restatement (tests/transform_oracle.c) on known cases."""
import numpy as np
import pytest

import rmse_exact as rx

F32 = np.float32


def _layer(blocks, vpb=8):
    """{block: [(voxel, d, observed)]} -> (idx, d, observed), unlisted voxels (0, unobserved)."""
    keys = list(blocks)
    idx = np.array(keys, np.int32).reshape(-1, 3)
    d = np.zeros((len(keys), vpb), F32)
    o = np.zeros((len(keys), vpb), bool)
    for k, b in enumerate(keys):
        for (v, dist, obs) in blocks[b]:
            d[k, v] = dist
            o[k, v] = obs
    return idx, d, o


# ---------------------------------------------------------------- RMSE rule, hand-derived answers
def test_rmse_shared_block_branches():
    gt = _layer({(0, 0, 0): [(0, 0.5, True), (1, 0.25, True), (2, 1.0, True), (3, 0.0, False),
                             (4, 0.1, True), (5, 0.0, False), (6, 0.3, True)]})
    test = _layer({(0, 0, 0): [(0, 0.75, True),     # e = 0.25
                               (1, -0.25, True),    # behind the surface: ignored
                               (2, 0.5, True),      # e = -0.5
                               (3, 0.2, True),      # gt unobserved: non-overlapping
                               (4, 0.3, False),     # test unobserved: non-overlapping
                               (5, 0.0, False),     # both unobserved: non-overlapping
                               (6, -0.0, True)]})   # -0.0 is not < 0: evaluated, e = -0.3
    r = rx.evaluate(gt, test)
    assert (r["num_evaluated_voxels"], r["num_ignored_voxels"], r["num_overlapping_voxels"],
            r["num_non_overlapping_voxels"]) == (3, 1, 4, 4)   # voxel 7: unobserved on both sides
    e = [F32(0.75) - F32(0.5), F32(0.5) - F32(1.0), F32(-0.0) - F32(0.3)]
    assert r["max_error"] == F32(0.5) and r["min_error"] == 0.0
    s = sum(float(F32(x * x)) for x in e)
    assert r["rmse"] == F32(np.sqrt(s / 3))


def test_rmse_nan_branches():
    gt = _layer({(0, 0, 0): [(0, 0.1, True), (1, np.nan, True), (2, 0.2, True)]})
    test = _layer({(0, 0, 0): [(0, 0.4, True), (1, 0.1, True), (2, np.nan, True)]})
    r = rx.evaluate(gt, test)
    # NaN test distance is not < 0: evaluated; a NaN error never becomes max_error, the sum turns NaN
    assert r["num_evaluated_voxels"] == 3 and r["num_ignored_voxels"] == 0
    assert r["max_error"] == F32(F32(0.4) - F32(0.1))
    assert np.isnan(r["rmse"]) and r["min_error"] == 0.0


def test_rmse_one_sided_blocks_and_empty():
    gt = _layer({(1, 0, 0): [(0, 0.1, True), (3, 0.1, True), (4, 0.0, False)],
                 (0, 0, 0): [(0, 0.1, False)]})
    test = _layer({(2, 0, 0): [(0, 0.1, True), (1, -1.0, True), (2, 0.0, False)],
                   (0, 0, 0): [(0, 0.2, True)]})
    r = rx.evaluate(gt, test)
    # test-only block: 2 observed; gt-only block: 2 observed; shared block: voxel 0 gt unobserved + 7 both
    assert r["num_non_overlapping_voxels"] == 2 + 2 + 8
    assert r["num_evaluated_voxels"] == 0 and r["num_overlapping_voxels"] == 0
    assert np.isnan(r["rmse"]) and r["max_error"] == 0.0
    empty = (np.zeros((0, 3), np.int32), np.zeros((0, 8), F32), np.zeros((0, 8), bool))
    r = rx.evaluate(empty, empty)
    assert np.isnan(r["rmse"]) and r["num_non_overlapping_voxels"] == 0


def test_rmse_observed_selectors():
    w = np.array([0, 1e-6, np.nextafter(F32(1e-6), F32(1)), 1], F32)
    assert rx.tsdf_observed(w).tolist() == [False, False, True, True]
    assert rx.esdf_observed(np.array([0, 1, 0.5], F32)).tolist() == [False, True, True]


# ---------------------------------------------------------------- transform restatement, known cases
def _box(vs, vps, seed=0):
    rs = np.random.RandomState(seed)
    idx = np.array([(i, j, k) for k in range(2) for j in range(2) for i in range(2)], np.int32)
    n = len(idx) * vps ** 3
    d = rs.uniform(0.05, 0.6, n).astype(F32).reshape(len(idx), -1)
    w = rs.uniform(0.5, 3.0, n).astype(F32).reshape(len(idx), -1)
    return vs, vps, idx, d, w


def test_transform_identity_is_a_no_op(oracle):
    import transform_oracle as to
    lay = _box(0.125, 8)
    out = to.transform_layer(oracle.Layer.from_blocks(*lay), np.array([1, 0, 0, 0, 0, 0, 0], F32)).export()
    assert np.array_equal(out[0], lay[2])   # the box is already in packed key order
    assert out[1].tobytes() == lay[3].tobytes() and out[2].tobytes() == lay[4].tobytes()


def test_transform_whole_voxel_translation_moves_blocks(oracle):
    import transform_oracle as to
    vs, vps, idx, d, w = _box(0.125, 8, seed=1)
    bs = float(F32(vs) * vps)
    out = to.transform_layer(oracle.Layer.from_blocks(vs, vps, idx, d, w),
                             np.array([1, 0, 0, 0, bs, 0, 0], F32)).export()
    keys = {tuple(b) for b in out[0].tolist()}
    assert keys == {tuple(b) for b in idx.tolist()} | {(2, j, k) for j in range(2) for k in range(2)}
    # voxel v of block b samples the centre of voxel v of block b - (1, 0, 0): the interpolation succeeds
    # (and returns that voxel exactly) where the voxel and its +1 neighbours lie inside the box; elsewhere an
    # old block keeps its voxel and a new block holds (0, 0)
    old = {tuple(c): s for s, c in enumerate(idx.tolist())}
    lin = np.arange(vps ** 3)
    loc = np.stack([lin % vps, (lin // vps) % vps, lin // (vps * vps)], -1)
    for k, b in enumerate(out[0].tolist()):
        src = (b[0] - 1, b[1], b[2])
        g = np.array(src)[None] * vps + loc                  # global voxel of the sample
        ok = np.all((g >= 0) & (g + 1 < 2 * vps), -1) if src in old else np.zeros(len(lin), bool)
        if src in old:
            assert out[1][k][ok].tobytes() == d[old[src]][ok].tobytes()
            assert out[2][k][ok].tobytes() == w[old[src]][ok].tobytes()
        if tuple(b) in old:
            assert out[1][k][~ok].tobytes() == d[old[tuple(b)]][~ok].tobytes()
            assert out[2][k][~ok].tobytes() == w[old[tuple(b)]][~ok].tobytes()
        else:
            assert not out[1][k][~ok].any() and not out[2][k][~ok].any()


def test_transform_failed_interpolation_keeps_old_voxel(oracle):
    import transform_oracle as to
    vs, vps, idx, d, w = _box(0.125, 8, seed=2)
    w[0, 0] = 0.0   # voxel (0, 0, 0) of block (0, 0, 0) unobserved
    T = np.array([1, 0, 0, 0, 0.01, 0, 0], F32)   # a sub-voxel shift: every sample needs its neighbours
    out = to.transform_layer(oracle.Layer.from_blocks(vs, vps, idx, d, w), T).export()
    k = [i for i, b in enumerate(out[0].tolist()) if b == [0, 0, 0]][0]
    # voxel 0 is moved to x - 0.01: below the first voxel centre of the layer: no interpolation, kept
    assert out[1][k][0] == d[0, 0] and out[2][k][0] == 0.0
    # voxel 1 interpolates between the unobserved voxel 0 and voxel 1: fails as well, kept
    assert out[1][k][1] == d[0, 1] and out[2][k][1] == w[0, 1]
    # voxel 2 interpolates between voxels 1 and 2: a new value
    assert out[1][k][2] != d[0, 2]
