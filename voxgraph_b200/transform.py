"""Float 6-DoF transforms: minkindr's QuatTransformationTemplate<float> (voxblox::Transformation, SURVEY.md
Appendix A.1) as the reference's front end uses it.

A transform is 7 float32 values [qw qx qy qz tx ty tz], the library's convention.  Every operation works in
float32 in the reference's order of operations (Eigen's quaternion product and _transformVector), so the
results are what the reference computes in float; exp keeps minkindr's double internals.  Host code only:
these run once per scan or per submap switch, never per point.
"""
import numpy as np

F32 = np.float32
IDENTITY = np.array([1, 0, 0, 0, 0, 0, 0], F32)
_EPS4 = np.finfo(np.float64).eps ** 0.25          # minkindr isLessThenEpsilons4thRoot (double)


def _rotate(q, v):
    """Eigen Quaternion::_transformVector: uv = 2 (vec x v); v + w uv + vec x uv."""
    w, x, y, z = q[0], q[1], q[2], q[3]
    uv = np.array([y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]], F32)
    uv = uv + uv
    c = np.array([y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0]], F32)
    return (v + w * uv) + c


def compose(A, B):
    """A * B."""
    A = np.asarray(A, F32); B = np.asarray(B, F32)
    aw, ax, ay, az = A[0], A[1], A[2], A[3]
    bw, bx, by, bz = B[0], B[1], B[2], B[3]
    q = np.array([aw * bw - ax * bx - ay * by - az * bz,
                  aw * bx + ax * bw + ay * bz - az * by,
                  aw * by + ay * bw + az * bx - ax * bz,
                  aw * bz + az * bw + ax * by - ay * bx], F32)
    return np.concatenate([q, A[4:] + _rotate(A, B[4:])]).astype(F32)


def inverse(T):
    """(R^T, -R^T t)."""
    T = np.asarray(T, F32)
    qi = np.array([T[0], -T[1], -T[2], -T[3]], F32)
    return np.concatenate([qi, -_rotate(qi, T[4:])]).astype(F32)


def exp(v6):
    """[t; rotation vector] -> T: the translation unchanged, the rotation RotationQuaternion::exp (Grassia)."""
    v = np.asarray(v6, F32)
    dx = v[3:]
    theta = float(np.sqrt(dx[0] * dx[0] + dx[1] * dx[1] + dx[2] * dx[2]))
    na = 0.5 + theta * theta * (1.0 / 48.0) if theta < _EPS4 else np.sin(theta * 0.5) / theta
    q = [np.cos(theta * 0.5), float(dx[0]) * na, float(dx[1]) * na, float(dx[2]) * na]
    return np.array([*q, v[0], v[1], v[2]], F32)


def log(T):
    """T -> [t; rotation vector] (Eigen's AngleAxis of the quaternion: angle 2 atan2(|vec|, |w|) in [0, pi])."""
    T = np.asarray(T, F32)
    vec = T[1:4]
    n = np.sqrt(vec[0] * vec[0] + vec[1] * vec[1] + vec[2] * vec[2])
    rv = np.zeros(3, F32)
    if n != 0:
        angle = F32(2) * np.arctan2(n, np.abs(T[0]))
        rv = vec / (-n if T[0] < 0 else n) * angle
    return np.concatenate([T[4:], rv]).astype(F32)


def gravity_align(T):
    """VoxgraphSubmapCollection::gravityAlignPose: zero roll and pitch of log(), then exp."""
    v = log(T)
    v[3] = 0
    v[4] = 0
    return exp(v)


def to_pose4(T):
    """[t, log()[5]] in float64: the 4-DoF pose a Pose4D node or a RelativePoseCostFunction reads off T."""
    v = log(T)
    return np.array([v[0], v[1], v[2], v[5]], np.float64)


def from_matrix(M):
    """4x4 homogeneous matrix -> T (Eigen's Quaternion from a rotation matrix, in double, then float)."""
    M = np.asarray(M, np.float64).reshape(4, 4)
    R = M[:3, :3]
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    if tr > 0:
        s = np.sqrt(tr + 1.0)
        w = 0.5 * s
        s = 0.5 / s
        q = [w, (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s]
    else:
        i = int(np.argmax(np.diag(R)))
        j = (i + 1) % 3; k = (j + 1) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        v = np.zeros(3)
        v[i] = 0.5 * s
        s = 0.5 / s
        v[j] = (R[j, i] + R[i, j]) * s
        v[k] = (R[k, i] + R[i, k]) * s
        q = [(R[k, j] - R[j, k]) * s, *v]
    return np.array([*q, *M[:3, 3]], F32)


def as_transform(pose, what="pose"):
    """A 7-vector [qw qx qy qz tx ty tz], a 4x4 homogeneous matrix or a 4-vector [x y z yaw] (zero roll and
    pitch) -> T.  A 7-vector whose quaternion is not of unit norm (|q|^2 off by more than 1e-3) is refused: it is
    most likely in another order, such as geometry_msgs' [x y z w]."""
    p = np.asarray(pose, np.float64)
    if p.shape == (4, 4):
        return from_matrix(p)
    if p.shape == (4,):
        return exp([p[0], p[1], p[2], 0.0, 0.0, p[3]])
    if p.shape == (7,):
        if abs(float(p[:4] @ p[:4]) - 1.0) > 1e-3:
            raise ValueError("%s: the quaternion [qw qx qy qz] = %s is not of unit norm" % (what, p[:4]))
        return p.astype(F32)
    raise ValueError("%s: expected [x y z yaw], [qw qx qy qz tx ty tz] or a 4x4 matrix, got shape %s"
                     % (what, p.shape))
