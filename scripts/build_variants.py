#!/usr/bin/env python
"""Builds tuning variants of libvoxgraph_b200.so into voxgraph_b200/variants/ (git-ignored, they
travel to the GPU box); scripts/tune_reg.sh times each one there."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from voxgraph_b200 import build as b  # noqa: E402

VARIANTS = {
    "b5": ["-DVGX_REG_THREADS=128", "-DVGX_REG_MIN_BLOCKS=5"],
    "b6": ["-DVGX_REG_THREADS=128", "-DVGX_REG_MIN_BLOCKS=6"],
    "b7": ["-DVGX_REG_THREADS=128", "-DVGX_REG_MIN_BLOCKS=7"],
    "b8": ["-DVGX_REG_THREADS=128", "-DVGX_REG_MIN_BLOCKS=8"],
    "t64_b12": ["-DVGX_REG_THREADS=64", "-DVGX_REG_MIN_BLOCKS=12"],
    "t64_b16": ["-DVGX_REG_THREADS=64", "-DVGX_REG_MIN_BLOCKS=16"],
    # ablations of the final kernel (results are wrong by construction: timing only)
    "x_nogram": ["-DVGX_X_NOGRAM=1"],
}

if __name__ == "__main__":
    out_dir = os.path.join(ROOT, "voxgraph_b200", "variants")
    os.makedirs(out_dir, exist_ok=True)
    names = sys.argv[1:] or list(VARIANTS)
    for name in names:
        out = os.path.join(out_dir, "libvgx_%s.so" % name)
        b.build(force=True, defines=VARIANTS[name], out=out)
        print("built", out)
