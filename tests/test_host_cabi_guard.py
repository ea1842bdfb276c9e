"""The C-ABI boundary keeps its contract by construction: every extern "C" function runs its body through
the one guard in csrc/vgx_internal.h (vgx_entry / vgx_entry_noctx), so no C++ exception crosses the
boundary, and a host allocation failure is VGX_ERR_NOMEM instead of std::terminate.  No CUDA here."""
import ctypes as C
import os
import re
import subprocess
import sys
import textwrap

import pytest

from collection_stream import field, varint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "voxgraph_b200", "csrc")

# trivial accessors that need no guard: no context state to set, nothing that can throw
TRIVIAL = {"vgx_device_count", "vgx_last_error", "vgx_ctx_stream", "vgx_launch_count",
           "vgx_tsdf_config_default", "vgx_esdf_config_default", "vgx_mesh_config_default",
           "vgx_registration_filter_default", "vgx_reg_config_default", "vgx_solver_options_default"}
# entry points whose bodies call other entry points; the inner calls only run their bodies
NESTED = {"vgx_ctx_destroy": {"vgx_comm_destroy"},
          "vgx_comm_init": {"vgx_comm_destroy"},
          "vgx_collection_load": {"vgx_collection_load_ex"},
          "vgx_mesh_ply": {"vgx_mesh_ply_ex"},
          "vgx_submap_finish_ex": {"vgx_submap_finish", "vgx_submap_extract_points"},
          "vgx_map_evaluate": {"vgx_project_map", "vgx_submap_transform", "vgx_evaluate_layers_rmse"},
          "vgx_mesh_build_combined": {"vgx_project_map", "vgx_mesh_build"}}


def _close(text, i, o, c):
    """Index just past the bracket that closes the one at text[i]."""
    depth = 0
    for k in range(i, len(text)):
        depth += (text[k] == o) - (text[k] == c)
        if depth == 0:
            return k + 1
    raise AssertionError("unbalanced %s" % o)


def code_only(text):
    """The source with comments removed and string and character literals emptied, so brackets balance."""
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'',
                  lambda m: "" if m.group(0)[0] == "/" else m.group(0)[0] * 2, text, flags=re.S)


def definitions():
    """{name: body} of every extern "C" definition under csrc/ (comments and literals blanked)."""
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if not f.endswith((".cu", ".cpp")):
            continue
        text = code_only(open(os.path.join(CSRC, f)).read())
        for m in re.finditer(r'extern ""[^;{(]*?\b(vgx_\w+)\s*\(', text):
            brace = _close(text, m.end() - 1, "(", ")")
            assert text[brace:].lstrip().startswith("{"), (f, m.group(1))
            start = text.index("{", brace)
            assert m.group(1) not in out, "defined twice: " + m.group(1)
            out[m.group(1)] = text[start + 1:_close(text, start, "{", "}") - 1]
    return out


def guarded(body):
    """The body is the one statement `return vgx_entry...(...);` (a void function drops the return)."""
    m = re.match(r"\s*(return\s+)?vgx_entry\w*\(", body)
    return bool(m) and body[_close(body, m.end() - 1, "(", ")"):].strip() == ";"


def test_every_entry_point_is_guarded():
    from voxgraph_b200 import _lib
    defs = definitions()
    assert set(defs) == set(_lib.EXPORTS)
    unguarded = sorted(n for n, b in defs.items() if n not in TRIVIAL and not guarded(b))
    assert unguarded == []
    for name, body in defs.items():
        calls = set(re.findall(r"\b(vgx_\w+)\s*\(", body)) & set(_lib.EXPORTS) - TRIVIAL - {name}
        assert calls <= NESTED.get(name, set()), (name, calls)
        assert all(guarded(defs[k]) for k in calls), name
        # the guard selects the device and vgx_submap_get looks submaps up; vgx_ctx_create selects its own
        assert "->find(" not in body, name
        assert "cudaSetDevice" not in body or name == "vgx_ctx_create", name


def minimal_collection(n_blocks):
    """A valid collection stream: one submap of n_blocks blocks (vps 2), each with a one-varint voxel_data."""
    vs, vps = 0.1, 2
    h = field(1, "d", vs) + field(2, "v", vps) + field(3, "v", 1)
    pose = field(1, "d", 0.0) + field(2, "d", 0.0) + field(3, "d", 0.0)
    rot = field(1, "d", 1.0) + field(2, "d", 0.0) + field(3, "d", 0.0) + field(4, "d", 0.0)
    sm = field(1, "v", 7) + field(2, "v", n_blocks) + field(3, "L", field(1, "L", pose) + field(2, "L", rot))
    blk = field(1, "v", vps) + field(2, "d", vs) + b"".join(field(3 + a, "d", 0.0) for a in range(3)) + \
        field(7, "v", 0)
    return varint(len(h)) + h + varint(len(sm)) + sm + (varint(len(blk)) + blk) * n_blocks


# Runs in a child: the address-space limit must not reach the test process.
CHILD = textwrap.dedent("""
    import ctypes as C, os, resource, sys
    sys.path.insert(0, sys.argv[1])
    from voxgraph_b200 import _lib
    lib = _lib.load()
    stream = open(sys.argv[2], "rb").read()
    n_scan = C.c_int(-1)
    out = (_lib.CollectionEntry * 1)()
    n = 4 << 20
    residuals, owner = (C.c_int32 * n)(), (C.c_int32 * n)()
    size = int(open("/proc/self/statm").read().split()[0]) * os.sysconf("SC_PAGE_SIZE")
    resource.setrlimit(resource.RLIMIT_AS, (size + (8 << 20), resource.getrlimit(resource.RLIMIT_AS)[1]))
    print(lib.vgx_collection_scan(stream, len(stream), 1, out, C.byref(n_scan)),
          lib.vgx_shard_constraints(2, n, residuals, None, owner))
""")


@pytest.fixture(scope="module")
def lib():
    from voxgraph_b200 import build, _lib
    build.build()
    return _lib.load()


def test_host_allocation_failure_is_nomem(lib, tmp_path):
    from voxgraph_b200 import _lib
    path = tmp_path / "stream.bin"
    path.write_bytes(minimal_collection(1 << 20))
    r = subprocess.run([sys.executable, "-c", CHILD, ROOT, str(path)], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0, r.stderr
    assert r.stdout.split() == [str(_lib.VGX_ERR_NOMEM)] * 2


def test_minimal_collection_scans(lib):
    """Without the limit, the stream above is a valid one-submap collection."""
    from voxgraph_b200 import _lib
    data = minimal_collection(1000)
    entries = (_lib.CollectionEntry * 1)()
    n = C.c_int()
    assert lib.vgx_collection_scan(data, len(data), 1, entries, C.byref(n)) == _lib.VGX_OK
    assert n.value == 1 and entries[0].id == 7 and entries[0].num_blocks == 1000
    assert entries[0].voxels_per_side == 2 and entries[0].voxel_size == pytest.approx(0.1)
