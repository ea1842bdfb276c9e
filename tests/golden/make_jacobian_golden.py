"""Generates tests/golden/pose_jacobians.json from the reference's own symbolic derivation.

Runs voxgraph/scripts/jacobians_xyz_yaw.py of a voxgraph checkout (sympy; import-only, prints
disabled), takes its T_eo and pose symbols, and lambdifies d(T_eo * o_r_oi)/d(params) —
the two 3x4 matrices hard-coded at registration_cost_function.cpp:214-227:
    python tests/golden/make_jacobian_golden.py <voxgraph checkout>/voxgraph/scripts/jacobians_xyz_yaw.py
"""
import contextlib
import io
import json
import os
import runpy
import sys

import numpy as np


def main(script):
    import sympy as sp
    with contextlib.redirect_stdout(io.StringIO()):
        ns = runpy.run_path(script)
    T_eo = ns["T_eo"]
    so = [ns[k] for k in ("x_o", "y_o", "z_o", "theta_o")]
    se = [ns[k] for k in ("x_e", "y_e", "z_e", "theta_e")]
    r = ns["o_r_oi"]
    rs = list(r.free_symbols)
    cols_o = [sp.simplify(sp.diff(T_eo, s) * r)[:3, 0] for s in so]
    cols_e = [sp.simplify(sp.diff(T_eo, s) * r)[:3, 0] for s in se]
    Mo = sp.Matrix.hstack(*cols_o)
    Me = sp.Matrix.hstack(*cols_e)
    # identify point symbols by name
    names = {str(s): s for s in rs}
    pt = [names[k] for k in sorted(names)]
    f_o = sp.lambdify(so + se + pt, Mo, "numpy")
    f_e = sp.lambdify(so + se + pt, Me, "numpy")
    rng = np.random.default_rng(4)
    cases = []
    for _ in range(24):
        ref = np.concatenate([rng.uniform(-1.5, 1.5, 3), rng.uniform(-3.0, 3.0, 1)])
        read = np.concatenate([rng.uniform(-1.5, 1.5, 3), rng.uniform(-3.0, 3.0, 1)])
        p = rng.uniform(-2.0, 2.0, 3); p[2] = rng.uniform(-0.5, 0.5)
        args = list(ref) + list(read) + list(p[:len(pt)])
        cases.append(dict(ref=ref.tolist(), read=read.tolist(), point=p.tolist(),
                          point_symbols=[str(s) for s in pt],
                          dTp_dref=np.asarray(f_o(*args), float).tolist(),
                          dTp_dread=np.asarray(f_e(*args), float).tolist()))
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pose_jacobians.json")
    json.dump(dict(source="voxgraph/scripts/jacobians_xyz_yaw.py", cases=cases), open(out, "w"), indent=1)
    print("wrote", out, len(cases), "cases; point symbols", [str(s) for s in pt])


if __name__ == "__main__":
    main(sys.argv[1])
