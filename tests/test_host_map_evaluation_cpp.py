"""The C++ mirror of MapEvaluation (voxgraph_b200/host/voxgraph_b200.hpp) compiles against the C-ABI with plain
g++; on a GPU it reports the same evaluation, bit for bit, as api.MapEvaluation on the protobuf layer fixture."""
import os
import subprocess

import numpy as np
import pytest

from support import compile_cpp_mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "layer_tsdf.bin")


def test_cpp_map_evaluation_compiles_and_refuses_cpu(tmp_path):
    import torch
    exe = compile_cpp_mirror(tmp_path, "map_evaluation_test.cpp")
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    p = subprocess.run([exe, FIXTURE], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout


@pytest.mark.gpu
def test_cpp_and_python_report_the_same_evaluation():
    import tempfile
    from voxgraph_b200 import api
    with tempfile.TemporaryDirectory() as tmp:
        import pathlib
        exe = compile_cpp_mirror(pathlib.Path(tmp), "map_evaluation_test.cpp")
        p = subprocess.run([exe, FIXTURE], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                           timeout=300)
    assert p.returncode == 0 and "MAPEVAL_OK" in p.stdout, p.stdout
    ctx = api.Context(0)
    me = api.MapEvaluation(ctx, FIXTURE, 900)
    with open(FIXTURE, "rb") as f:
        nb = ctx.layer_load(901, f.read())
    ev = me.evaluate([901], np.array([[1, 0, 0, 0, 0, 0, 0]], np.float32))
    ctx.close()
    r = ev.reconstruction
    bits = lambda x: "%08x" % int(np.float32(x).view(np.uint32))
    line = "MAPEVAL_OK blocks=%d rmse=%s max=%s eval=%d ign=%d ovl=%d non=%d term=%d T=%s" % (
        nb, bits(r.rmse), bits(r.max_error), r.num_evaluated_voxels, r.num_ignored_voxels,
        r.num_overlapping_voxels, r.num_non_overlapping_voxels, ev.summary.termination,
        "".join(bits(t) for t in ev.T_ground_truth__reading))
    assert line in p.stdout, (line, p.stdout)
    assert r.num_overlapping_voxels > 0
