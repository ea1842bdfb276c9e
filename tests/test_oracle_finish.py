"""The finishSubmap harness (tests/finish_exact.py) against the oracle on the CPU: ESDF, relevant
voxels, surface OBB and isosurface vertices over the layer matrix, filter and ESDF configurations,
the dense-noise layers that once hung the oracle, block-order independence, and planted faults that
the comparisons must catch."""
import numpy as np
import pytest

import finish_exact as fx
from finish_exact import ESDF_CASES, FILTERS, MATRIX


def _grid_and_layer(oracle, vs, vps, idx, d, w):
    return fx.Grid(vs, vps, idx, d, w), oracle.Layer.from_blocks(vs, vps, idx, d, w)


def check_layer(oracle, vs, vps, idx, d, w, min_w=1.0, max_d=0.3, esdf_cfg=None):
    """Harness == oracle bit for bit; returns (harness isosurface dict, Jacobi sweeps, oracle sweeps)."""
    g, L = _grid_and_layer(oracle, vs, vps, idx, d, w)
    cfg = esdf_cfg or {}
    e, ob, sw = fx.esdf(g, **{k[:-2] if k.endswith("_m") else k: v for k, v in cfg.items()})
    eo, obo, swo = oracle.generate_esdf(L, oracle.esdf_config(**cfg) if cfg else None)
    fx.assert_bits(eo, e, "esdf distance")
    fx.assert_bits(obo, ob, "esdf observed")
    assert sw <= fx.sweep_bound(cfg.get("max_distance_m", 2.0), vs)[1]
    xyz, dd, ww, (ok, mn, mx) = fx.relevant(g, min_w, max_d)
    fx.assert_points(oracle.find_relevant_voxels(L, min_w, max_d), (xyz, dd, ww), "relevant")
    ok_o, mn_o, mx_o = oracle.surface_obb(L, min_w, max_d)
    assert ok == ok_o
    if ok:
        fx.assert_bits(mn_o, mn, "obb min"); fx.assert_bits(mx_o, mx, "obb max")
    iso = fx.isosurface(g, min_w)
    xo, do_, wo, blk = oracle.find_isosurface_vertices(L, min_w)
    fx.assert_points((xo, do_, wo), (iso["xyz"], iso["distance"], iso["weight"]), "isosurface")
    assert np.array_equal(blk, iso["blocks"])
    # the float32 interpolation against the float64 trilinear value, where the bound's first-order
    # derivation holds (offset error E <= 2^-8: not at the far ends of the index range)
    small = fx.U * (3 * np.abs(iso["xyz"] * g.bsi).max(1, initial=0) * vps + 2 * vps + 4) <= 2.0 ** -8
    for k, b in (("d64", "bound_d"), ("w64", "bound_w")):
        got = (iso["distance"] if k == "d64" else iso["weight"]).astype(np.float64)
        assert np.all(np.abs(got - iso[k])[small] <= iso[b][small]), k
    return iso, sw, swo


@pytest.mark.parametrize("case", range(len(MATRIX)), ids=[m[0] for m in MATRIX])
def test_harness_equals_oracle(oracle, case):
    check_layer(oracle, *MATRIX[case][1])


def test_crafted_field_reaches_its_edges(oracle):
    """The crafted field hits every branch it is built for: midpoint vertices, t = 1 vertices on a voxel
    centre, and bucket keys exactly on half boundaries at both signs, with even integer parts (where
    llround and rint differ)."""
    vs, vps, idx, d, w = fx.layer((0.25, 8), "straddle", "crafted")
    iso = fx.isosurface(fx.Grid(vs, vps, idx, d, w), 1.0)
    x = iso["cand"].astype(np.float64) * (1.0 / np.float64(np.float32(0.125)))
    half = np.abs(x - np.floor(x)) == 0.5
    even = half & (np.floor(np.abs(x)) % 2 == 0)
    assert (even & (x > 0)).any() and (even & (x < 0)).any()
    assert not np.array_equal(fx.round_half_away(x[even]), np.rint(x[even]).astype(np.int64))
    check_layer(oracle, vs, vps, idx, d, w)


@pytest.mark.parametrize("case", range(len(FILTERS)), ids=[f[0] for f in FILTERS])
def test_filters_harness_equals_oracle(oracle, case):
    vs, vps, idx, d, w, mw, md = FILTERS[case][1]
    iso, _, _ = check_layer(oracle, vs, vps, idx, d, w, min_w=mw, max_d=md)
    if mw == 0.1 and w[0, 0] == np.float32(0.1):
        # relevant in double (0.1f > 0.1), not a cube corner in float (0.1f <= 0.1f)
        assert len(iso["xyz"]) == 0
        assert len(fx.relevant(fx.Grid(vs, vps, idx, d, w), mw, md)[0]) > 0


@pytest.mark.parametrize("case", range(len(ESDF_CASES)), ids=[c[0] for c in ESDF_CASES])
def test_esdf_configs_harness_equals_oracle(oracle, case):
    name, lay, cfg = ESDF_CASES[case]
    _, sw, swo = check_layer(oracle, *lay, esdf_cfg=cfg)
    if name == "5m-at-0.05":
        assert sw >= 99        # 99 sweeps change something: the device runs at least 100
    if name == "max-reached-exactly":
        e = fx.esdf(fx.Grid(*lay), max_distance=1.0, min_distance=0.3)[0].reshape(8, 8, 8)
        assert np.all(e[:, :, 2] == 0.75) and np.all(e[:, :, 3] == 2.0)    # 1.0 is not below max_distance


def test_esdf_edge_join_propagates_through_the_edge(oracle):
    """The plane lies in the first group only; the second group, joined along one block edge, is
    reached through edge and corner neighbours only."""
    vs, vps, idx, d, w = fx.layer((0.25, 8), "edge", "plane")
    d = d.copy(); d[2:] = 0.6                        # the second group carries no surface
    e, ob, _ = fx.esdf(fx.Grid(vs, vps, idx, d, w), max_distance=4.0, default_distance=4.0)
    assert (e[2:] < 4.0).any()


@pytest.mark.parametrize("vps", [16, 32])
def test_dense_noise_oracle_returns(oracle, vps):
    """One block of random-sign noise: more distinct buckets than the oracle's bucket set once held
    (it was sized from 4096 per block, whatever the vps), and more vertices than its wrapper's output."""
    vs, vps, idx, d, w = fx.noise_layer(0.05, vps, (1, 1, 1), seed=3)
    iso, _, _ = check_layer(oracle, vs, vps, idx, d, w)
    assert len(iso["xyz"]) > 4096


def test_block_order_independence(oracle):
    """Permuting the blocks leaves the ESDF of every block index unchanged, and the relevant voxels
    unchanged as a set, ordered by the new slot order."""
    vs, vps, idx, d, w = fx.layer((0.2, 16), "checker", "tilted")
    perm = np.random.RandomState(5).permutation(len(idx))
    g0, L0 = _grid_and_layer(oracle, vs, vps, idx, d, w)
    g1, L1 = _grid_and_layer(oracle, vs, vps, idx[perm], d[perm], w[perm])
    e0 = oracle.generate_esdf(L0)[0]; e1 = oracle.generate_esdf(L1)[0]
    fx.assert_bits(e0[perm], e1, "esdf under a permutation")
    fx.assert_bits(fx.esdf(g1)[0], e1, "harness esdf under a permutation")
    x0, d0, _ = oracle.find_relevant_voxels(L0)
    x1, d1, _ = oracle.find_relevant_voxels(L1)
    assert sorted(map(tuple, x0.tolist())) == sorted(map(tuple, x1.tolist()))
    bsi = g1.bsi
    slot_of = {tuple(b): k for k, b in enumerate(idx[perm].tolist())}
    slots = [slot_of[tuple(b)] for b in np.floor(x1 * bsi).astype(int).tolist()]
    assert slots == sorted(slots)


def test_planted_faults_are_caught(oracle):
    """One ESDF voxel one ulp off, one vertex dropped, and two bucket winners swapped each fail."""
    vs, vps, idx, d, w = fx.layer((0.2, 16), "box", "sphere")
    g, L = _grid_and_layer(oracle, vs, vps, idx, d, w)
    e = fx.esdf(g)[0]
    eo = oracle.generate_esdf(L)[0]
    k = np.nonzero(eo.reshape(-1) > 0.5)[0][7]
    e1 = e.copy().reshape(-1); e1[k] = np.nextafter(e1[k], np.float32(np.inf))
    with pytest.raises(AssertionError):
        fx.assert_bits(eo, e1.reshape(e.shape), "esdf")
    iso = fx.isosurface(g, 1.0)
    ref = oracle.find_isosurface_vertices(L, 1.0)[:3]
    drop = [np.delete(a, 11, axis=0) for a in (iso["xyz"], iso["distance"], iso["weight"])]
    with pytest.raises(AssertionError):
        fx.assert_points(ref, drop, "isosurface")
    # swap the winner of the first shared bucket with its runner-up
    keys, win = iso["keys"], iso["winners"]
    packed = [tuple(k) for k in keys.tolist()]
    first = {}
    swapped = None
    for c, kk in enumerate(packed):
        if kk in first and first[kk] in set(iso["kept"].tolist()):
            swapped = (first[kk], c)
            break
        first.setdefault(kk, c)
    assert swapped is not None
    kept = iso["kept"].copy(); kept[kept == swapped[0]] = swapped[1]
    ok, d32, w32 = fx.interp(g, iso["cand"][kept])[:3]
    assert ok.all()
    with pytest.raises(AssertionError):
        fx.assert_points(ref, (iso["cand"][kept], d32, w32), "isosurface")
