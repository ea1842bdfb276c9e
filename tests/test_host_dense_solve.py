"""The backward-error harness of tests/solve_exact.py, checked on the oracle's plain float64 Cholesky,
and the dispatch sizes and rank rule it assumes, read from solve.cu."""
import os
import re

import numpy as np
import pytest

import solve_exact as SX

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxgraph_b200", "csrc")


def _solve_src():
    with open(os.path.join(CSRC, "solve.cu")) as f:
        return f.read()


def _oracle_first_step(oracle, spec, radius, jacobi):
    og = SX.oracle_graph(oracle, spec)
    ok, _, g, H = og.eval()
    assert ok
    rc, s = og.solve(oracle.solver_options(max_num_iterations=1, initial_trust_region_radius=radius,
                                           jacobi_scaling=jacobi, **SX.FORCED))
    assert rc == 0 and s.num_successful_steps == 1
    return H, g, og.poses()


@pytest.mark.parametrize("n", [4, 12, 32, 64])
@pytest.mark.parametrize("radius", [1e4, 1.0, 1e-3])
@pytest.mark.parametrize("jacobi", [0, 1])
def test_oracle_step_passes_and_perturbed_steps_fail(oracle, n, radius, jacobi):
    """The oracle's recovered first step passes the bound.  Where the step is comparable to the
    poses (radius >= 1), an error of 2^-44 relative in one component (fast_rsqrt with one Newton
    step) and a solve that dropped one off-diagonal term of A both fail it.  Under heavy damping
    the step is ~1e-4 of the poses and the recovery term ulp(x1) hides relative errors below ~1e-12."""
    spec = SX.make_graph(n, anchor="interleaved", seed=n)
    H, g, x1 = _oracle_first_step(oracle, spec, radius, jacobi)
    ratio, (A, b, y, scale) = SX.step_ratio(H, g, spec.x0, x1, spec.free, radius, jacobi)
    assert ratio < 1, ratio
    if radius < 1:
        return
    _, delta = SX.recover_step(spec.x0, x1, spec.free, scale)
    yf = np.asarray(y, np.float64)
    # one component off by 2^-44 relative, in the row where the bound is tightest
    aL = np.abs(np.linalg.cholesky(A))
    base = SX.gamma_c(n) * SX.U * (aL @ (aL.T @ np.abs(yf)))
    i = int(np.argmax(np.abs(np.diag(A) * yf) / (base + np.abs(A) @ delta)))
    yp = y.copy()
    yp[i] *= 1 + np.longdouble(2.0 ** -44)
    assert SX.backward_ratio(A, b, yp, delta) > 1
    # the largest off-diagonal contribution |A_ij y_j| left out of the solve
    off = np.abs(A * yf[None, :])
    off[np.diag_indices_from(off)] = 0
    i, j = np.unravel_index(int(np.argmax(off)), off.shape)
    Ad = A.copy()
    Ad[i, j] = Ad[j, i] = 0.0
    assert SX.backward_ratio(A, b, np.linalg.solve(Ad, b), delta) > 1


def test_rank_threshold_separates_gauge_freedom_from_anchored_chains(oracle):
    """Right-looking float64 Cholesky of the oracle's J^T J.  Gauge-free graphs (no constant node)
    have a 4-dimensional null space; the first pivot that is not clearly positive must be at
    least 3 orders of magnitude below the rank tolerance.  Anchored chains, with and without loop
    closures, must have every pivot at least 3 orders above it."""
    tau = SX.RANK_TOL
    worst_null, worst_anchored = 0.0, np.inf
    for k, (F, loops) in enumerate([(8, True), (16, False), (40, True), (64, False), (64, True)]):
        spec = SX.make_graph(4 * F, anchor="none", loops=loops, seed=100 + k)
        ok, _, _, H = SX.oracle_graph(oracle, spec).eval()
        p = SX.relative_pivots(H, stop=tau * 1e3)
        assert p[-1] < tau * 1e3, "gauge-free J^T J factored without a small pivot"
        worst_null = max(worst_null, abs(p[-1]))
    for k, (F, loops) in enumerate([(64, False), (250, False), (120, True)]):
        spec = SX.make_graph(4 * F, anchor="first", loops=loops, seed=200 + k, info=SX.INFO_ODOM)
        ok, _, _, H = SX.oracle_graph(oracle, spec).eval()
        Hf = H[np.ix_(spec.free, spec.free)]
        p = SX.relative_pivots(Hf, stop=tau * 1e3)
        assert len(p) == Hf.shape[0] and p[-1] >= tau * 1e3, "anchored chain has a pivot near the tolerance"
        worst_anchored = min(worst_anchored, p.min())
    assert worst_null <= tau * 1e-3, worst_null
    assert worst_anchored >= tau * 1e3, worst_anchored


def test_dispatch_sizes_follow_the_source():
    """The GPU size lists straddle solve.cu's one dispatch: the last LM size solved in shared memory
    and the first on the cooperative grid.  The covariances always factor on the cooperative grid;
    their sizes cross a CH_NB panel edge.  Moving a limit in solve.cu fails this until the sizes move."""
    src = _solve_src()
    assert len(re.findall(r"static int chol_dispatch\(", src)) == 1
    assert len(re.findall(r"cudaOccupancyMaxActiveBlocksPerMultiprocessor\(&per_sm, chol_coop_kernel,", src)) == 1
    assert len(re.findall(r"cudaLaunchCooperativeKernel\(", src)) == 1
    assert re.findall(r"chol_dispatch\(c, n, (true|false),", src) == ["false", "true"], \
        "the covariances (first) must not take the shared-memory solver, the LM (second) may"
    m = re.findall(r"const size_t smem_chol_bytes = sizeof\(double\) \* \(\(size_t\)\(n \+ 1\) \* \(n \+ 2\) / 2 \+ n \+ 2\);", src)
    assert len(m) == 1, "the shared-memory solver's footprint changed"
    m = re.findall(r"const bool use_smem_chol = n > 0 && n <= (\d+) && smem_chol_bytes <= (\d+) \* 1024;", src)
    assert len(m) == 1, "the shared-memory solver's size test changed"
    n_cap, kib = int(m[0][0]), int(m[0][1])

    def fits(n):
        return n <= n_cap and 8 * ((n + 1) * (n + 2) // 2 + n + 2) <= kib * 1024

    smem_max = max(n for n in range(4, 4096, 4) if fits(n))
    coop_min = smem_max + 4
    assert not fits(coop_min)
    assert (smem_max, coop_min) == (SX.SMEM_MAX_N, SX.COOP_MIN_N)
    assert smem_max in SX.LM_SIZES and coop_min in SX.LM_SIZES
    m = re.findall(r"#define CH_NB (\d+)", src)
    assert len(m) == 1
    panel_edge = 8 * int(m[0])   # n = 256: the last unknown closes chol_coop_kernel's 8th panel
    for n in (panel_edge - 4, panel_edge, panel_edge + 4):
        assert n in SX.COV_SIZES
    assert all(n % 4 == 0 for n in SX.LM_SIZES + SX.COV_SIZES)


def test_rank_tolerance_is_the_kernels():
    src = _solve_src()
    m = re.findall(r"#define VGX_COV_RANK_TOL (\S+)", src)
    assert len(m) == 1 and float(m[0]) == SX.RANK_TOL
