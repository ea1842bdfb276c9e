"""The C++ mirror of cblox's collection file I/O (LoadSubmapCollection / SaveSubmapCollection in
voxgraph_b200/host/voxgraph_b200.hpp) compiles against the C-ABI with plain g++; on a GPU a fixture
loaded and saved through it comes back byte for byte."""
import os
import subprocess

import pytest

from support import compile_cpp_mirror

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "collection_unpacked.bin")


def test_cpp_collection_io_compiles_and_refuses_cpu(tmp_path):
    import torch
    exe = compile_cpp_mirror(tmp_path, "collection_io_test.cpp")
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu test")
    p = subprocess.run([exe, FIXTURE, str(tmp_path / "out.bin")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 2 and "no CPU fallback" in p.stdout


@pytest.mark.gpu
def test_cpp_collection_io_on_gpu(tmp_path):
    exe = compile_cpp_mirror(tmp_path, "collection_io_test.cpp")
    out = tmp_path / "out.bin"
    p = subprocess.run([exe, FIXTURE, str(out)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=300)
    assert p.returncode == 0 and "COLLECTION_IO_OK submaps=3" in p.stdout, p.stdout
    assert out.read_bytes() == open(FIXTURE, "rb").read()
