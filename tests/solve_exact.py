"""Backward-error checks of the dense pose-graph solves (test support; importable without a GPU).

The Levenberg-Marquardt step and the edge covariances go through hand-written Cholesky kernels
(solve.cu: chol_solve_smem_kernel, chol_coop_kernel + lm_step_kernel, chol_coop_kernel + cov_column_kernel).
Converged poses cannot pin them: LM corrects a step that is wrong by 1e-6 relative in its next
iteration.  What a correct float64 Cholesky solve guarantees, whatever the conditioning, is a small
backward error (Higham, Accuracy and Stability of Numerical Algorithms, Thm 10.4):

    (A + dA) y = b,   |dA| <= gamma_{3n+1} |L| |L^T|,   so   |b - A y| <= gamma_{3n+1} |L| |L^T| |y|

per row, with L any float64 Cholesky factor of A (only magnitudes are used).  The checks below
compute that residual in long double and report its largest ratio to the bound.

The device does not return the LM step itself, only the poses after it.  With every step forced
to be accepted, the poses after one iteration are fl(x0 + d) with d = fl(-y * scale); for yaws in
(-pi, pi) normalize_angle is the identity (2 pi floor(.) is exactly 0), so d^ = x1 - x0 lies within
ulp(x1) + u |d| of d in each component.  That is carried as a known perturbation of y^ = -d^ / scale,
and the bound gains |A| delta.  The recovery is sharp when |d| is comparable to |x|, so the graph
builders start the free poses up to a metre away from the poses the measurements describe.
"""
import numpy as np

U = 2.0 ** -53                 # unit roundoff of float64
SLACK = 8                      # fast_rsqrt (a few ulps) and the restated A (fma on the diagonal)
RANK_TOL = 1e-10               # solve.cu VGX_COV_RANK_TOL: pivot <= tol * H_kk is rank deficient
FRAME_ID = 0x80000000          # api.FRAME_NODE_ID_BASE: reference-frame node 0
INFO_ODOM = np.diag([1.0, 1.0, 2500.0, 2500.0])

# Dispatch edges of solve.cu (tests/test_host_dense_solve.py derives them from the source):
# the LM factors in shared memory up to n = 232 and on the cooperative grid from 236; the
# covariances always use the cooperative grid (252 | 256 | 260 cross one of its panel edges).
SMEM_MAX_N = 232
COOP_MIN_N = 236
LM_SIZES = [4, 8, 12, 28, 32, 36, 124, 128, 132, 228, 232, 236, 252, 256, 260, 796, 1000]
COV_SIZES = [4, 20, 32, 36, 64, 68, 252, 256, 260, 796]

# every step accepted, nothing terminates early: the poses returned after k iterations are
# x0 plus k steps
FORCED = dict(min_relative_decrease=-1e300, parameter_tolerance=0.0, function_tolerance=0.0)


def gamma_c(n):
    return 3 * n + 1 + SLACK


class Spec:
    """A relative-pose graph: node ids (ascending, which is the device's node order), initial poses,
    constant flags and edges (node index a, node index b, t_obs[3], yaw_obs, information 4x4)."""

    def __init__(self, ids, x0, constant, edges):
        self.ids = [int(i) for i in ids]
        self.x0 = np.asarray(x0, np.float64)
        self.constant = np.asarray(constant, bool)
        self.edges = edges
        assert self.ids == sorted(self.ids)

    @property
    def N(self):
        return len(self.ids)

    @property
    def free(self):
        """Indices of the free unknowns in the 4N parameter vector: the reduced order of graph.cu."""
        return np.array([4 * i + k for i in range(self.N) if not self.constant[i] for k in range(4)], int)

    @property
    def n(self):
        return len(self.free)


def _rel(pa, pb):
    c, s = np.cos(pa[3]), np.sin(pa[3])
    d = pb[:3] - pa[:3]
    y = pb[3] - pa[3]
    return np.array([c * d[0] + s * d[1], -s * d[0] + c * d[1], d[2]]), y - 2 * np.pi * np.floor((y + np.pi) / (2 * np.pi))


def _info(rng):
    """A random SPD information matrix with coupled axes (dense sqrt-information)."""
    Lm = np.diag([1.0, 1.0, 10.0, 20.0] * rng.uniform(0.5, 2.0, 4)) + np.tril(rng.normal(0, 0.3, (4, 4)), -1)
    return Lm @ Lm.T


def make_graph(n, anchor="first", loops=True, seed=0, untouched=False, info=None):
    """A relative-pose graph with n free unknowns (n % 4 == 0).

    anchor: "first" (node 0 constant), "interleaved" (node 0, every 7th node and the last node
    constant, so the reduced offsets have gaps), "frame" (every submap node free, anchored by
    absolute-pose constraints from a constant reference-frame node) or "none" (gauge-free: a
    4-dimensional null space).  untouched: one of the free nodes has no constraint at all.
    loops: chain plus loop closures, or the chain alone.  Some chain edges are also given in the
    opposite direction and one edge is repeated.  info: a fixed information matrix, else a random
    dense one per edge.
    """
    assert n % 4 == 0 and n > 0
    rng = np.random.default_rng(seed)
    F = n // 4
    constant = []
    if anchor == "first":
        constant = [True] + [False] * F
    elif anchor == "interleaved":
        i = 0
        while constant.count(False) < F:
            constant.append(i % 7 == 0)
            i += 1
        constant.append(True)
    elif anchor in ("frame", "none"):
        constant = [False] * F
    else:
        raise ValueError(anchor)
    ids = list(range(len(constant)))
    if anchor == "frame":
        ids.append(FRAME_ID)
        constant.append(True)
    N = len(ids)
    gt = np.concatenate([rng.uniform(-3, 3, (N, 2)), rng.uniform(-0.5, 0.5, (N, 1)),
                         rng.uniform(-1.2, 1.2, (N, 1))], 1)
    if anchor == "frame":
        gt[-1] = 0.0
    x0 = gt + np.concatenate([rng.uniform(-0.8, 0.8, (N, 2)), rng.uniform(-0.2, 0.2, (N, 1)),
                              rng.uniform(-0.25, 0.25, (N, 1))], 1)
    x0[np.array(constant)] = gt[np.array(constant)]
    x0[:, 3] = np.clip(x0[:, 3], -1.45, 1.45)
    loose = None
    if untouched:
        loose = int(np.flatnonzero(~np.array(constant))[F // 2])
    nodes = [i for i in range(N) if ids[i] != FRAME_ID and i != loose]
    edges = []

    def edge(a, b):
        t, y = _rel(gt[a], gt[b])
        t = t + rng.normal(0, 0.01, 3)
        y = y + rng.normal(0, 0.002)
        edges.append((a, b, t, y, info if info is not None else _info(rng)))

    for k in range(len(nodes) - 1):
        a, b = nodes[k], nodes[k + 1]
        if k % 5 == 3:
            a, b = b, a
        edge(a, b)
        if k % 6 == 1:
            edge(b, a)
        if k == 2:
            edge(a, b)
    if loops:
        for _ in range(max(1, len(nodes) // 2)):
            a, b = rng.choice(len(nodes), 2, replace=False)
            if abs(int(a) - int(b)) >= 2:
                edge(nodes[a], nodes[b])
    if anchor == "frame":
        for k in (0, len(nodes) // 2, len(nodes) - 1):
            edge(N - 1, nodes[k])
    spec = Spec(ids, x0, constant, edges)
    assert spec.n == n
    return spec


def pose_graph(api, ctx, spec):
    """The spec as an api.PoseGraph (absolute-pose constraints for edges from the frame node)."""
    pg = api.PoseGraph(ctx)
    for i, nid in enumerate(spec.ids):
        if nid >= FRAME_ID:
            pg.addReferenceFrameNode(api.ReferenceFrameNodeConfig(nid - FRAME_ID, spec.x0[i], bool(spec.constant[i])))
        else:
            pg.addSubmapNode(api.SubmapNodeConfig(nid, spec.x0[i], set_constant=bool(spec.constant[i])))
    for (a, b, t, y, info) in spec.edges:
        m = np.array([*t, y])
        if spec.ids[a] >= FRAME_ID:
            pg.addAbsolutePoseConstraint(api.AbsolutePoseConstraintConfig(spec.ids[a] - FRAME_ID, spec.ids[b], m, info))
        else:
            pg.addRelativePoseConstraint(api.RelativePoseConstraintConfig(spec.ids[a], spec.ids[b], m, info))
    return pg


def oracle_graph(oracle, spec):
    og = oracle.Graph()
    for i, nid in enumerate(spec.ids):
        og.add_node(nid, spec.x0[i], constant=bool(spec.constant[i]))
    for (a, b, t, y, info) in spec.edges:
        og.add_relative(spec.ids[a], spec.ids[b], t, y, oracle.sqrt_information(info))
    return og


# ------------------------------------------------------------------ LM restatement
def lm_system(H, g, free, radius, jacobi, scale=None, min_diag=1e-6, max_diag=1e32):
    """float64 restatement of lm_build_kernel + lm_persist_kernel on the reduced problem:
    A = S H S + diag(clamp(S^2 H_kk) / radius) and b = S g.  scale: the Jacobi scale kept from
    iteration 0 (None: compute it from this H, as on the first iteration)."""
    Hf = H[np.ix_(free, free)]
    D = np.diag(Hf).copy()
    if scale is None:
        scale = 1.0 / (1.0 + np.sqrt(D)) if jacobi else np.ones(len(free))
    A = (scale[:, None] * scale[None, :]) * Hf
    d = np.clip(scale * scale * D, min_diag, max_diag)
    lm = np.sqrt(d / radius)
    A[np.diag_indices_from(A)] += lm * lm
    return A, scale * g[free], scale


def recover_step(x0, x1, free, scale):
    """y^ = -(x1 - x0) / scale over the free unknowns, and delta >= |y^ - y| componentwise."""
    ld = np.longdouble
    a0 = np.asarray(x0, np.float64).reshape(-1)[free]
    a1 = np.asarray(x1, np.float64).reshape(-1)[free]
    yaw = free % 4 == 3
    assert np.all(np.abs(a1[yaw]) < 3.0), "a yaw left (-3, 3): normalize_angle is not the identity"
    d = a1.astype(ld) - a0.astype(ld)
    y = -d / scale.astype(ld)
    # x1 = fl(x0 + d): ulp(x1); d = fl(y * scale): u |d|; the long double difference and quotient
    delta = (np.spacing(np.abs(a1)) + 2.0 * U * np.abs(d.astype(np.float64))) / scale * (1 + 1e-9)
    return y, delta


def _max_ratio(r, bound):
    """max |r| / bound; an entry with a zero bound (a block of A decoupled from the right-hand side
    or column) must have a zero residual."""
    r = np.abs(r).astype(np.float64)
    zero = bound == 0
    if np.any(r[zero] != 0):
        return np.inf
    return float(np.max(r[~zero] / bound[~zero]))


def backward_ratio(A, b, y, delta=None, extra=None):
    """max_i |b - A y|_i / (c u (|L||L^T||y|)_i + (|A| delta)_i + extra_i), residual in long double.
    extra: a known perturbation of A times |y| (e.g. an uncertain damping term)."""
    ld = np.longdouble
    n = len(b)
    aL = np.abs(np.linalg.cholesky(A))
    ay = np.abs(np.asarray(y, np.float64))
    bound = gamma_c(n) * U * (aL @ (aL.T @ ay))
    if delta is not None:
        bound = bound + np.abs(A) @ delta
    if extra is not None:
        bound = bound + extra
    r = np.asarray(b, ld) - np.dot(np.asarray(A, ld), np.asarray(y, ld))
    return _max_ratio(r, bound)


def model_cost_change(H, g, free, scale, y):
    """Ceres' model cost change -(s^T gs + 1/2 s^T Hs s) of the scaled step s = -y."""
    y = np.asarray(y, np.float64)
    Hs = (scale[:, None] * scale[None, :]) * H[np.ix_(free, free)]
    return float(y @ (scale * g[free]) - 0.5 * y @ (Hs @ y))


def step_ratio(H, g, x0, x1, free, radius, jacobi, scale=None):
    """Backward-error ratio of the LM step x0 -> x1, plus the (A, b, y^, scale) it used."""
    A, b, scale = lm_system(H, g, free, radius, jacobi, scale)
    y, delta = recover_step(x0, x1, free, scale)
    return backward_ratio(A, b, y, delta), (A, b, y, scale)


# ------------------------------------------------------------------ covariances
def covariance_ratio(Hf, X, cols):
    """Columns X of Hf^-1 (X[:, k] for unknown cols[k]): max |Hf X - E| / (c u |L||L^T||X|)."""
    ld = np.longdouble
    n = Hf.shape[0]
    aL = np.abs(np.linalg.cholesky(Hf))
    E = np.zeros((n, len(cols)), ld)
    E[np.asarray(cols), np.arange(len(cols))] = 1
    R = np.dot(np.asarray(Hf, ld), np.asarray(X, ld)) - E
    bound = gamma_c(n) * U * (aL @ (aL.T @ np.abs(X)))
    return _max_ratio(R, bound)


def relative_pivots(H, stop):
    """Right-looking float64 Cholesky of H: the pivots d_k / H_kk, up to and including the first
    that is below `stop` (after it the factorisation has no meaning)."""
    A = np.array(H, np.float64)
    h = np.diag(A).copy()
    out = []
    for k in range(A.shape[0]):
        d = A[k, k]
        out.append(d / h[k] if h[k] > 0 else 0.0)
        if not out[-1] >= stop:
            break
        l = A[k + 1:, k] / np.sqrt(d)
        A[k + 1:, k + 1:] -= np.outer(l, l)
    return np.array(out)
