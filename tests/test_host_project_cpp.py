"""The C++ mirror of the combined-mesh service (ProjectMap / GenerateCombinedMesh / SaveCombinedMesh in
voxgraph_b200/host/voxgraph_b200.hpp) compiles against the C-ABI with plain g++; on a GPU it writes the
same PLY bytes as api.save_combined_mesh for the submaps of a collection fixture."""
import os
import subprocess

import pytest

from support import compile_cpp_mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "collection_unpacked.bin")


def test_cpp_combined_mesh_compiles_and_refuses_cpu(tmp_path):
    import torch
    exe = compile_cpp_mirror(tmp_path, "combined_mesh_test.cpp")
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    p = subprocess.run([exe, FIXTURE, str(tmp_path / "out.ply")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout


@pytest.mark.gpu
def test_cpp_and_python_write_the_same_combined_ply(tmp_path):
    from voxgraph_b200 import api
    exe = compile_cpp_mirror(tmp_path, "combined_mesh_test.cpp")
    out = tmp_path / "cpp.ply"
    p = subprocess.run([exe, FIXTURE, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=300)
    assert p.returncode == 0 and "COMBINED_OK submaps=3" in p.stdout, p.stdout
    ctx = api.Context(0)
    ids, poses = api.load_submap_collection(ctx, FIXTURE)
    py = tmp_path / "py.ply"
    api.save_combined_mesh(ctx, str(py), ids, poses)
    ctx.close()
    assert out.read_bytes() == py.read_bytes()
    assert "blocks=0" not in p.stdout
