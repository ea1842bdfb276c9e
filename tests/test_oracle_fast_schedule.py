"""The race-aware model of the Fast schedule (tests/fast_schedule.py) pinned to the oracle: every sequential
order it simulates equals the oracle's mode-1 integration bit for bit, every sequential outcome lies in the
interleaving search's set, the checker accepts every oracle outcome (threaded runs included) and rejects
outcomes that no interleaving can produce."""
import itertools

import numpy as np
import pytest

import fast_schedule as fs
import tsdf_exact as tx

FACTORS, MS, RES = fs.FACTORS, fs.MS, fs.RES


def _oracle_run(oracle, sc, order, threads=0):
    """The oracle's mode-1 integration of the scene's points in `order` -> (stats tuple, layer)."""
    layer = oracle.Layer(sc.vs, sc.vps)
    cfg = oracle.tsdf_config(**dict(sc.kw, max_consecutive_ray_collisions=sc.m))
    pts = sc.pts[list(order)]
    if threads:
        st = oracle.tsdf_integrate_mt(layer, cfg, sc.T, pts, threads)
    else:
        st = oracle.tsdf_integrate(layer, cfg, sc.T, pts)
    return (st.rays_valid, st.rays_cast, st.voxel_updates, st.blocks_allocated), layer.export()


def _micro(oracle, name, vs, vps, factor, sensor):
    T, pts, cfg = fs.micro_scene(name, vs, factor, sensor)
    sc = fs.Scene(oracle, vs, vps, T, pts, **cfg)
    fs.assert_micro_property(sc, name, sensor)
    assert sc.decodable()
    return sc


def _all_micro(oracle, res=RES, sensors=("origin", "negative")):
    for (vs, vps), sensor, factor, name in itertools.product(res, sensors, FACTORS, fs.MICRO_NAMES):
        yield name, sensor, _micro(oracle, name, vs, vps, factor, sensor)


def test_simulate_equals_oracle_every_order(oracle):
    """Each micro scene, every permutation of its points, every collision limit, factor and sensor at
    one resolution (all three for the default order)."""
    n = 0
    for name, sensor, sc in _all_micro(oracle):
        for m in MS:
            sc.m = m
            orders = itertools.permutations(range(len(sc.pts))) if sc.vs == 0.1 else [range(len(sc.pts))]
            for order in orders:
                out = sc.simulate(order)
                st, lay = _oracle_run(oracle, sc, order)
                assert st == sc.stats(out), (name, sensor, m, order)
                tx.assert_layers_bit_equal(lay, sc.layer(sc.updates(out, order)))
                n += 1
    assert n > 1000


def test_simulate_equals_oracle_random_orders(oracle):
    rs = np.random.RandomState(7)
    for _ in range(60):
        sc = fs.random_scene(oracle, rs)
        for _ in range(3):
            order = rs.permutation(len(sc.pts))
            out = sc.simulate(order)
            st, lay = _oracle_run(oracle, sc, order)
            assert st == sc.stats(out)
            tx.assert_layers_bit_equal(lay, sc.layer(sc.updates(out, order)))


def test_sequential_outcomes_are_reachable(oracle):
    """Every sequential order's outcome is among the interleavings; some micro scenes have more than one
    reachable outcome (the races the device can show)."""
    multi = total = 0
    for name, sensor, sc in _all_micro(oracle, res=[(0.1, 16)]):
        for m in MS:
            sc.m = m
            reach = sc.reachable()
            canon = {sc.canonical(o) for o in reach}
            for order in itertools.permutations(range(len(sc.pts))):
                out = sc.simulate(order)
                assert tuple(out[i] for i in sc.valid) in reach, (name, sensor, m, order)
                assert sc.canonical(out) in canon
            total += 1
            multi += len(canon) > 1
    print("micro scenes with more than one reachable outcome: %d of %d" % (multi, total))
    assert multi > 0.3 * total


def test_checker_accepts_oracle_outcomes(oracle):
    """Sequential orders of micro and random scenes, and the threaded oracle (atomic exchanges)."""
    for name, sensor, sc in _all_micro(oracle, res=[(0.05, 8)]):
        for m in MS:
            sc.m = m
            reach = {sc.canonical(o) for o in sc.reachable()}
            for order in itertools.permutations(range(len(sc.pts))):
                st, lay = _oracle_run(oracle, sc, order)
                info = sc.check(lay, st)
                assert info["decoded"] in reach
    rs = np.random.RandomState(11)
    for k in range(80):
        sc = fs.random_scene(oracle, rs)
        order = rs.permutation(len(sc.pts))
        st, lay = _oracle_run(oracle, sc, order, threads=4 if k % 2 else 0)
        sc.check(lay, st)


def _mutants(sc, out):
    """(kind, layer, stats) of hand-made changes to one sequential outcome."""
    ups = sc.updates(out)
    for i, (c, p) in out.items():
        r = sc.rays[i]
        if c and p < len(r.seq):
            for q in (p - 1, p + 1):                     # the break moved by one voxel
                if 0 <= q <= len(r.seq):
                    o2 = dict(out); o2[i] = (True, q)
                    yield "break moved", sc.layer(sc.updates(o2)), sc.stats(o2)
            blk = sc.block(r.seq[p])                     # the break voxel's block allocated
            if blk not in sc.blocks_of(ups):
                yield "break block", sc.layer(ups, [blk]), sc.stats(out, [blk])
        if not c and len(sc.slots[r.slot]) == 1:         # a de-duplicated ray cast (whole or cut)
            for q in {len(r.seq), min(sc.m, len(r.seq))}:
                o2 = dict(out); o2[i] = (True, q)
                yield "skip cast", sc.layer(sc.updates(o2)), sc.stats(o2)
        if p >= 2:                                       # one update dropped or applied twice
            k = (i, (p - 1) // 2)
            drop = [x for x in ups if x != k]
            st = sc.stats(out)
            yield "dropped", sc.layer(drop), st[:2] + (st[2] - 1, len(sc.blocks_of(drop)))
            yield "duplicated", sc.layer(ups + [k]), st[:2] + (st[2] + 1, st[3])


def test_checker_rejects_unreachable_mutations(oracle):
    """Every mutation of a sequential outcome whose decoded outcome no interleaving produces is rejected
    (a layer the decoder cannot read is never produced), and every kind is exercised.  Most are caught
    by rules (a)-(f) alone; a break moved within a run of voxels that other rays also visited needs the
    exact search."""
    seen, by_rules = {}, {}
    extra = [("marker_block", "origin", _micro(oracle, "marker_block", 0.05, 8, f, "origin")) for f in FACTORS]
    for name, sensor, sc in itertools.chain(_all_micro(oracle, res=[(0.05, 8), (0.1, 16)]), extra):
        for m in MS:
            sc.m = m
            reach = {sc.canonical(o) for o in sc.reachable()}
            for order in itertools.permutations(range(len(sc.pts))):
                for kind, lay, st in _mutants(sc, sc.simulate(order)):
                    try:
                        dec = sc.check(lay, st)["decoded"]
                    except AssertionError:
                        by_rules[kind] = by_rules.get(kind, 0) + 1
                    else:
                        if dec in reach:
                            continue             # reachable after all: not a provable error
                        with pytest.raises(AssertionError):
                            sc.check(lay, st, reach)
                    seen[kind] = seen.get(kind, 0) + 1
    print("rejected mutations:", seen, "of them by rules (a)-(f):", by_rules)
    assert set(seen) == {"break moved", "break block", "skip cast", "dropped", "duplicated"}
    assert all(by_rules.get(k) == v for k, v in seen.items() if k != "break moved")
    assert by_rules["break moved"] > 0


def test_marker_rule(oracle):
    """(-1, 0, 0) and (17190, -1, 0) hash to the sets' empty marker ~0: at the identity, a point whose
    start cell is (-1, 0, 0) is never cast, and a ray's first visit of voxel (-1, 0, 0) is a collision
    (with m = 0 a ray ends there before updating it)."""
    assert fs.any_index_hash(-1, 0, 0) == fs.MARKER == fs.any_index_hash(17190, -1, 0)
    vs = 0.1
    T, pts, cfg = fs.micro_scene("marker", vs, 2, "origin")
    for m in (0, 1):
        sc = fs.Scene(oracle, vs, 16, T, pts, **dict(cfg, max_consecutive_ray_collisions=m))
        out = sc.simulate()
        assert out[1] == (False, 0)
        r = sc.rays[0]
        k = r.seq.index((-1, 0, 0))
        assert out[0] == ((True, k) if m == 0 else (True, len(r.seq)))
        st, lay = _oracle_run(oracle, sc, range(len(pts)))
        assert st == sc.stats(out)
        tx.assert_layers_bit_equal(lay, sc.layer(sc.updates(out)))
