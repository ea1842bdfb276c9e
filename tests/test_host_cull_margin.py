"""The cull margin of reg_unit_may_hit, on its float32 restatement (tests/reduce_exact.py).

The reduce kernel skips a 32-point unit when the transformed bounding sphere, widened by a margin for
the float error of the per-point transform, touches no existing block.  The fused sums are exact only
if no skipped unit holds a point whose block index (computed as stage A computes it) exists.  Block
indices are monotone in the coordinate, so that holds when every point's transform lies inside the
float box (centre - R, centre + R) the kernel tests; the tests below check that box directly."""
import os
import re

import numpy as np

import reduce_exact as RX

F32 = np.float32
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxgraph_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_restatement_constants_match_the_kernel():
    """The restatement's margin terms, S and n1 are the kernel's: a change to reg_unit_may_hit or
    VGX_COORD_EPS has to be made in tests/reduce_exact.py too, where the checks below see it."""
    src = _src("registration.cu")
    body = src[src.index("reg_unit_may_hit("):]
    body = body[:body.index("\n}\n")]
    m = re.findall(r"const float R = b\.w \+ \(b\.w \* \(2\.0f \* n1 \+ (0x1p-\d+)f\) \+ S \* (0x1p-\d+)f\);", body)
    assert len(m) == 1, "reg_unit_may_hit's radius expression changed"
    assert float.fromhex(m[0][0]) == float(RX.MARGIN_R)
    assert float.fromhex(m[0][1]) == float(RX.MARGIN_S)
    assert "const float n1 = fabsf(P.qw * P.qw + P.qz * P.qz - 1.0f);" in body
    assert ("const float S = ((fabsf(b.x) + fabsf(b.y)) + (fabsf(b.z) + 3.0f * b.w)) +\n"
            "                  ((fabsf(P.tx) + fabsf(P.ty)) + fabsf(P.tz));") in body
    m = re.findall(r"#define VGX_COORD_EPS (\S+)f", _src("registration.cuh"))
    assert len(m) == 1 and F32(float(m[0])) == RX.COORD_EPS


def _pose(rng, t_max, yaw):
    return np.array([*rng.uniform(-t_max, t_max, 2), rng.uniform(-50, 50), yaw]).astype(F32).astype(np.float64)


def _units(rng, n_units, c_max):
    """float32 units: centres up to c_max from the origin, radii 0 and 1e-7 .. 3 m, points on the
    sphere surface rounded to float32 (so they sit up to an ulp of c_max off it)."""
    c = np.concatenate([rng.uniform(-c_max, c_max, (n_units, 2)), rng.uniform(-50, 50, (n_units, 1))], 1)
    c = c.astype(F32).astype(np.float64)
    r = np.where(rng.random(n_units) < 0.2, 0.0, 10.0 ** rng.uniform(-7, 0.5, n_units))
    d = rng.normal(size=(n_units, 32, 3))
    d /= np.linalg.norm(d, axis=2, keepdims=True)
    return (c[:, None, :] + r[:, None, None] * d).astype(F32)


def _box_misses(P, X, b, margin_s=None):
    """Points of units whose transform leaves the kernel's cull box (float32), per unit."""
    p = RX.transform(P, X.reshape(-1, 3)).reshape(X.shape)
    _, _, L, H, _ = RX.cull_box(P, b, margin_s=margin_s)
    out = ((p < L[:, None, :]) | (p > H[:, None, :])).any((1, 2))
    return out, p


def test_cull_box_holds_every_point():
    """100 000 float32 units at 1 m to 10 km from the origin, translations of the same size, yaws
    over the whole range (and 0, +-pi, the series branch): every point's transform lies in the
    kernel's box, so its block index lies between the box's.  The fuzz reaches units whose float
    error needs more than S * 2^-24 (the same check with that margin fails) and shows how much of
    the S * 2^-16 margin the worst unit uses."""
    rng = np.random.default_rng(0)
    bsi = F32(1.0) / (F32(0.2) * F32(16))
    worst = 0.0
    over_24 = 0
    missed_24 = 0
    units = 0
    for trial in range(20):
        t_max = [1.0, 100.0, 2000.0, 1.0e4][trial % 4]
        yaw_r, yaw_e = rng.uniform(-np.pi, np.pi, 2)
        if trial % 4 == 1:
            yaw_r = [0.0, float(F32(np.pi)), -float(F32(np.pi)), 5e-5, 1e-9][trial // 4]
        P = RX.pose_block(_pose(rng, t_max, yaw_r), _pose(rng, t_max, yaw_e))
        X = _units(rng, 5000, t_max)
        b = RX.unit_bounds(X, np.ones(X.shape[:2], F32))
        miss, p = _box_misses(P, X, b)
        assert not miss.any(), (trial, np.flatnonzero(miss)[:5])
        c, R, L, H, S = RX.cull_box(P, b)
        blk = RX.block_index(p.reshape(-1, 3), bsi).reshape(p.shape)
        assert (blk >= RX.block_index(L, bsi)[:, None, :]).all() and (blk <= RX.block_index(H, bsi)[:, None, :]).all()
        # how much of the S term each unit needs: the largest per-axis distance from the transformed
        # centre beyond the radius and n-terms of R, relative to S
        n1 = float(np.abs(P["qw"] * P["qw"] + P["qz"] * P["qz"] - F32(1.0)))
        r = b[:, 3].astype(np.float64)
        dev = np.abs(p.astype(np.float64) - c[:, None, :].astype(np.float64)).max((1, 2))
        need = (dev - (r + r * (2.0 * n1 + float(RX.MARGIN_R)))) / S.astype(np.float64)
        worst = max(worst, float(need.max()))
        over_24 += int((need > 2.0 ** -24).sum())
        missed_24 += int(_box_misses(P, X, b, margin_s=2.0 ** -24)[0].sum())
        units += len(b)
    print("cull margin: %d units, worst need %.3g S (margin %.3g S), %d need more than 2^-24 S, "
          "%d would be dropped at 2^-24" % (units, worst, float(RX.MARGIN_S), over_24, missed_24))
    assert units == 100000
    assert over_24 > 0 and missed_24 > 0, "the fuzz never needed more than S * 2^-24"
    assert worst < float(RX.MARGIN_S)


def test_culling_scene_contributors_are_live(oracle):
    """On the culling-edge scene of tests/test_gpu_reduce_exact.py (reduce_exact.cull_problem_scenes,
    both pairs at the same poses), every point the oracle finds a correspondence for lies in a unit the
    restated cull test keeps live; the GPU test then shows the fused sums include all of them."""
    bsi = oracle.Layer(RX.CULL_VS, RX.CULL_VPS).block_size_inv
    x, scenes = RX.cull_problem_scenes(bsi)
    for (ref, read, P, sc) in scenes:
        assert RX.check_pose_block(oracle, x[ref], x[read]) == P
        layer = oracle.Layer.from_blocks(RX.CULL_VS, RX.CULL_VPS, sc["block_idx"], sc["distance"], sc["weight"])
        ok, r, jr, je = oracle.reg_evaluate(layer, sc["xyz"], sc["d"], sc["w"], x[ref], x[read])
        assert ok
        contrib = (r != 0) | (np.abs(jr).sum(1) > 0)
        mh, mh0, hits = RX.cull_report(P, sc)
        live_pt = np.repeat(mh, 32)[:len(r)]
        assert contrib.sum() > 300
        assert not (contrib & ~live_pt).any()
        assert not (hits & ~mh).any()
        assert mh.any() and (~mh).any() and (mh & ~mh0).any()
