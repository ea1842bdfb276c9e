"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol
include/voxgraph_b200.h declares, and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os

import pytest

import support

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from voxgraph_b200 import build, _lib
    build.build()
    return _lib.load()


def test_header_symbols_exported(lib):
    from voxgraph_b200 import _lib
    declared = support.header_functions()
    assert len(declared) >= 30
    assert declared == set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name


# the header typedef of every ctypes.Structure in voxgraph_b200/_lib.py
HEADER_STRUCTS = {"TsdfConfig": "vgx_tsdf_config", "TsdfStats": "vgx_tsdf_stats",
                  "RegistrationFilter": "vgx_registration_filter", "RegConfig": "vgx_reg_config",
                  "EsdfConfig": "vgx_esdf_config", "SolverOptions": "vgx_solver_options",
                  "SolverSummary": "vgx_solver_summary", "CollectionEntry": "vgx_collection_entry",
                  "MeshConfig": "vgx_mesh_config", "VoxelEvaluationDetails": "vgx_voxel_evaluation_details",
                  "MapEvaluationResult": "vgx_map_evaluation", "CloudLayout": "vgx_cloud_layout"}


def test_struct_layouts_match_header(tmp_path):
    """Every ctypes mirror in _lib.py against the C compiler's view of include/voxgraph_b200.h (size and
    every field offset), and every VGX_ constant of _lib.py (status codes, layer selectors, profiling
    slots) against its value in the header."""
    from voxgraph_b200 import _lib
    constants = {n: v for n, v in vars(_lib).items() if n.startswith("VGX_") and isinstance(v, int)}
    assert "VGX_SLOT_EVAL" in constants and "VGX_PROFILE_SLOTS" in constants
    support.check_struct_layouts(tmp_path, _lib, HEADER_STRUCTS, constants=constants)
    assert C.sizeof(_lib.TsdfConfig) == 14 * 4 and C.sizeof(_lib.TsdfStats) == 5 * 8
    assert C.sizeof(_lib.CollectionEntry) == 44
    assert C.sizeof(_lib.VoxelEvaluationDetails) == 48
    assert C.sizeof(_lib.CloudLayout) == 36
    assert C.sizeof(_lib.MeshConfig) == 4 and _lib.MeshConfig.min_weight.offset == 0


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from voxgraph_b200 import _lib, api
    h = C.c_void_p()
    assert lib.vgx_device_count() == 0
    assert lib.vgx_ctx_create(0, C.byref(h)) == _lib.VGX_ERR_CUDA
    with pytest.raises(api.VgxError):
        api.Context(0)


def test_product_does_not_import_oracle():
    """The oracle is test infrastructure: nothing under voxgraph_b200/ may reference it."""
    pkg = os.path.join(ROOT, "voxgraph_b200")
    for dirpath, _, files in os.walk(pkg):
        if os.path.basename(dirpath) == "build":
            continue
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "vg_oracle" not in txt and "import oracle" not in txt and \
                    "from oracle" not in txt, os.path.join(dirpath, f)
