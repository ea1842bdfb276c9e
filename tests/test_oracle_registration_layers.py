"""The oracle's registration lookup (vgo_reg_evaluate) against the dense-grid interpolator of
tests/finish_exact.py over the finishSubmap layer matrix, on the CPU.

At identity poses with distance 0 and weight 1 every residual is 0 - interp: the oracle's residual must
equal 0 - float(finish_exact.interp) bit for bit (so +0.0 where the interpolation gives either zero), the two correspondence masks must agree, the float32 value must
lie within interp_bound of the float64 trilinear value wherever the bound's first-order derivation holds,
and no far point (tests/registration_layers.py: blocks 2^21 away from real ones, and just beyond both ends
of the index range) may find a correspondence.  This pins the reference the GPU tests compare with.

B1 evaluation order: the harness and vgo_reg_evaluate both evaluate each row of B1 * distances left to
right, (((d0 - d2) - d4) + d6) and so on, as written in registration_cost_function.h:73-81; the bit-for-bit
comparison below would fail if either used another order.
"""
import numpy as np
import pytest

import finish_exact as fx
import registration_layers as RL
from finish_exact import MATRIX

IDENTITY = np.zeros(4)


def evaluate(oracle, layer, xyz):
    """vgo_reg_evaluate at identity poses, distance 0, weight 1 -> (hit mask, residuals).  A missing
    correspondence costs NaN, which no interpolated value is."""
    n = len(xyz)
    ok, r, _, _ = oracle.reg_evaluate(layer, xyz, np.zeros(n, np.float32), np.ones(n, np.float32),
                                      IDENTITY, IDENTITY, no_correspondence_cost=float("nan"),
                                      jacobians=False)
    assert ok
    return ~np.isnan(r), r


def check_layer(oracle, vs, vps, idx, d, w, seed=0):
    P = RL.points(vs, vps, idx, d, w, seed=seed)
    g, xyz = P["grid"], P["xyz"]
    L = oracle.Layer.from_blocks(vs, vps, idx, d, w)
    hit, r = evaluate(oracle, L, xyz)
    ok, d32, _, d64, _, bound, _ = fx.interp(g, xyz)
    bad = np.nonzero(hit != ok)[0]
    assert bad.size == 0, ("correspondence masks differ", P["kind"][bad[0]], xyz[bad[0]].tolist(), bool(hit[bad[0]]))
    want = 0.0 - d32[ok].astype(np.float64)      # (distance - interp) * weight: +0.0 where interp is +-0.0
    got = r[ok]
    bad = np.nonzero(want.view(np.uint64) != got.view(np.uint64))[0]
    assert bad.size == 0, ("residual != -interp", P["kind"][ok][bad[0]], float(got[bad[0]]), float(want[bad[0]]))
    # float32 against float64 trilinear, where E <= 2^-8 (finish_exact module docstring)
    small = fx.U * (3 * np.abs(P["block"]).max(1) * vps + 2 * vps + 4) <= 2.0 ** -8
    sel = ok & small
    assert np.all(np.abs(d32[sel].astype(np.float64) - d64[sel]) <= bound[sel])
    assert not hit[P["far"]].any(), "a far point found a correspondence"
    return P, hit


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_oracle_lookup_equals_harness(oracle, case):
    vs, vps, idx, d, w = MATRIX[case][1]
    P, hit = check_layer(oracle, vs, vps, idx, d, w, seed=case)
    kinds = set(P["kind"].tolist())
    assert "far_end" in kinds
    if len(idx):
        assert {"centre", "corner", "face", "plane", "random", "far_alias"} <= kinds
        assert hit.any() and (~hit & ~P["far"]).any()
        # far points whose 21-bit key is a real block's: the case the device's hash probe must refuse
        assert RL.aliases(P["block"][P["far"]], idx).sum() >= len(idx)


def test_vps2_points_wrap_into_the_lower_block(oracle):
    """At vps 2 every voxel touches a block face: about half of all centre points have their base
    corner in the lower neighbour block on some axis (the `wrap` branch)."""
    vs, vps, idx, d, w = fx.layer((0.05, 2), "box", "tilted")
    P = RL.points(vs, vps, idx, d, w)
    c = P["xyz"][P["kind"] == "centre"]
    g = P["grid"]
    b = RL.contain_block(c, g.bsi)
    v = np.floor((((c - (b.astype(np.float32) * g.bs).astype(np.float32)).astype(np.float32) * g.vsi)
                  + fx._EPS)).astype(np.int64)
    # a centre lies exactly on its voxel's centre: the base corner is that voxel, and it is voxel 0
    # (the wrap's precondition) on some axis for 7 of 8 voxels
    assert np.mean((v == 0).any(1)) > 0.8
    ok = fx.interp(g, P["xyz"])[0]
    assert ok.any()
    check_layer(oracle, vs, vps, idx, d, w)


def test_checker_and_corner_layouts_miss_through_corners(oracle):
    """Checkerboard and corner-joined layouts: points whose containing block exists but whose octet
    reaches into a missing block have no correspondence in both implementations."""
    for lay in ("checker", "corner"):
        vs, vps, idx, d, w = fx.layer((0.2, 16), lay, "plane")
        P, hit = check_layer(oracle, vs, vps, idx, d, w)
        exist = np.isin(RL._key(P["block"]), RL._key(idx)) & RL.in_range(P["block"])
        assert (exist & ~hit).sum() > 100


def test_planted_lookup_faults_are_caught(oracle):
    """A residual one ulp off, a correspondence dropped, and a far point answered with the aliased
    block's value each fail the comparison."""
    vs, vps, idx, d, w = fx.layer((0.25, 8), "box", "crafted")
    P = RL.points(vs, vps, idx, d, w)
    g, xyz = P["grid"], P["xyz"]
    L = oracle.Layer.from_blocks(vs, vps, idx, d, w)
    hit, r = evaluate(oracle, L, xyz)
    ok, d32 = fx.interp(g, xyz)[:2]
    k = np.nonzero(ok & (d32 != 0))[0][5]
    r1 = r.copy(); r1[k] = np.nextafter(r1[k], np.inf)
    assert (r1[ok].view(np.uint64) != (0.0 - d32[ok].astype(np.float64)).view(np.uint64)).any()
    hit1 = hit.copy(); hit1[k] = False
    assert (hit1 != ok).any()
    # the aliasing lookup: the far point evaluated at its aliased (real) position does hit
    far = np.nonzero(P["far"] & RL.aliases(P["block"], idx))[0]
    assert len(far)
    j = far[0]
    shifted = P["block"][j] - idx[np.nonzero(RL._key(idx) == RL._key(P["block"][j:j + 1])[0])[0][0]]
    assert set(np.abs(shifted).tolist()) <= {0, RL.ALIAS}
