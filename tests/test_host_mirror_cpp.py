"""The C++ host mirror (voxgraph_b200/host/voxgraph_b200.hpp) compiles against the C-ABI with plain
g++ (the reference is C++: this is the layer a maintainer links); on a GPU it must reproduce the
closed-form plane residuals, solve, and integrate a scan."""
import subprocess

import pytest

from support import compile_cpp_mirror


def test_cpp_mirror_compiles_and_refuses_cpu(tmp_path):
    import torch
    exe = compile_cpp_mirror(tmp_path, "host_mirror_test.cpp")
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout


@pytest.mark.gpu
def test_cpp_mirror_on_gpu(tmp_path):
    exe = compile_cpp_mirror(tmp_path, "host_mirror_test.cpp")
    p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert p.returncode == 0 and "HOST_MIRROR_OK" in p.stdout, p.stdout
