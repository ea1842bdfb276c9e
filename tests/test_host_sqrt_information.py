"""The square-root information factor both host mirrors hand to vgx_graph_set_relative_edges comes from one place,
vgx_sqrt_information: api.sqrt_information_matrix and the C++ SqrtInformation (driver tests/cpp/
sqrt_information_test.cpp, plain g++ against the library) give the same bits, reject the same matrices with the
reference's messages, and keep the factors the C++ mirror computed before the rule moved into the library.
No GPU needed."""
import subprocess

import numpy as np
import pytest

from support import compile_cpp_mirror
from voxgraph_b200 import api

_v, _w = np.array([1.0, 2.0, 0.5, -1.0]), np.array([0.3, -1.0, 2.0, 0.5])
MATRICES = {
    "diagonal": np.diag([2.0, 3.0, 5.0, 7.0]),
    "dense_spd": np.array([[4.0, 1.2, -0.6, 0.3], [1.2, 3.0, 0.5, -0.2], [-0.6, 0.5, 2.5, 0.7],
                           [0.3, -0.2, 0.7, 1.8]]),
    "rank2_psd": np.outer(_v, _v) + np.outer(_w, _w),
    "height": np.diag([0.0, 0.0, 2500.0, 0.0]),          # AbsolutePoseConstraint with information zz only
    "indefinite": np.array([[1.0, 2.0, 0.0, 0.0], [2.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]),
}
LLT_ERROR = ("The square root of the information matrix could not be computed, make sure it is symmetric and "
             "positive definite")
LDLT_ERROR = "The information matrix must be positive semi-definite"
_Z = "0000000000000000"
_DIAG = ["3ff6a09e667f3bcd", _Z, _Z, _Z, _Z, "3ffbb67ae8584caa", _Z, _Z, _Z, _Z, "4001e3779b97f4a8", _Z, _Z, _Z, _Z,
         "40052a7fa9d2f8ea"]
# (matrix, allow_semi_definite) -> the 16 factor entries' IEEE-754 bits as the C++ mirror's own LLT / LDLT code
# computed them, or the error message
EXPECTED = {
    ("diagonal", 0): _DIAG,
    ("diagonal", 1): _DIAG,
    ("dense_spd", 0): ["4000000000000000", _Z, _Z, _Z, "3fe3333333333333", "3ff9ff3656bdf346", _Z, _Z,
                       "bfd3333333333333", "3fdac8e2a6f24076", "3ff7eb47374661bc", _Z, "3fc3333333333333",
                       "bfc6d88515ecbe84", "3fe18bc9acf923c4", "3ff33bb7fe0296fb"],
    ("dense_spd", 1): ["4000000000000000", _Z, _Z, _Z, "3fe3333333333333", "3ff9ff3656bdf346", _Z, _Z,
                       "bfd3333333333333", "3fdac8e2a6f24075", "3ff7eb47374661bc", _Z, "3fc3333333333333",
                       "bfc6d88515ecbe84", "3fe18bc9acf923c4", "3ff33bb7fe0296fb"],
    ("rank2_psd", 0): LLT_ERROR,
    ("rank2_psd", 1): ["3e50000000000000", "3fe854134e7cbd5f", "3fe6e5b7d16657e1", _Z, _Z, "4001e3779b97f4a8", _Z, _Z,
                       _Z, "bfdc9f25c5bfedda", "400019853f3bf5ca", _Z, "be40000000000000", "bff1e3779b97f4a8", _Z, _Z],
    ("height", 0): LLT_ERROR,
    ("height", 1): [_Z] * 10 + ["4049000000000000"] + [_Z] * 5,
    ("indefinite", 0): LLT_ERROR,
    ("indefinite", 1): LDLT_ERROR,
}


def _python(info, semi):
    try:
        return ["%016x" % b for b in api.sqrt_information_matrix(info, semi).reshape(-1).view(np.uint64)]
    except ValueError as e:
        return str(e)


@pytest.fixture(scope="module")
def cpp(tmp_path_factory):
    """-> {(name, allow_semi_definite): bits or message} from the C++ mirror."""
    exe = compile_cpp_mirror(tmp_path_factory.mktemp("sqrt_information"), "sqrt_information_test.cpp")
    keys = list(EXPECTED)
    stdin = "".join("%d %s\n" % (semi, " ".join(float(x).hex() for x in MATRICES[name].reshape(-1)))
                    for name, semi in keys)
    p = subprocess.run([exe], input=stdin, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True)
    out = {}
    for key, line in zip(keys, p.stdout.splitlines()):
        kind, rest = line.split(" ", 1)
        out[key] = rest.split() if kind == "ok" else rest
    assert len(out) == len(keys), p.stdout
    return out


@pytest.mark.parametrize("key", list(EXPECTED), ids=["%s-%s" % (n, "ldlt" if s else "llt") for n, s in EXPECTED])
def test_both_mirrors_give_the_reference_factor(cpp, key):
    name, semi = key
    assert cpp[key] == EXPECTED[key]
    assert _python(MATRICES[name], semi) == EXPECTED[key]

