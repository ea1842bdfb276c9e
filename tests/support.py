"""Helpers that two or more test modules share.  pytest does not collect this module (it collects
test_*.py only); a helper that one module uses stays in that module.

A GPU module takes the context fixture with `from support import ctx  # noqa: F401`: the fixture is
module-scoped, so each module that imports it gets a context of its own.  The synthetic room `world` is
imported the same way."""
import atexit
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import finish_exact as fx
from collection_stream import field, varint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32
IDENTITY = np.array([1, 0, 0, 0, 0, 0, 0], F32)   # T [qw qx qy qz tx ty tz]


@pytest.fixture(scope="module")
def ctx():
    from voxgraph_b200 import api
    c = api.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def world():
    """The 30 m x 30 m synthetic room the integration tests scan."""
    from voxgraph_b200 import synth
    return synth.make_world(3, size_xy=(30.0, 30.0), n_clutter=40, n_walls=4)


def same_bits(exp, got, what):
    """Bit-equal arrays, NaN equal to NaN whatever its payload."""
    exp = np.asarray(exp); got = np.asarray(got)
    assert exp.shape == got.shape, (what, exp.shape, got.shape)
    if exp.dtype == np.float32:
        ne, ng = np.isnan(exp), np.isnan(got)
        assert np.array_equal(ne, ng), (what, "NaN positions")
        exp = np.where(ne, 0, exp).astype(F32); got = np.where(ng, 0, got).astype(F32)
        fx.assert_bits(exp, got, what)
    else:
        bad = np.nonzero(exp != got)
        assert bad[0].size == 0, (what, "first difference at", bad[0][:1], exp[bad][:3], got[bad][:3])


def exists(ctx, sid):
    """Whether submap sid exists; any error other than VGX_ERR_NOT_FOUND fails."""
    from voxgraph_b200 import _lib, api
    try:
        ctx.submap_info(sid)
        return True
    except api.VgxError as e:
        assert e.code == _lib.VGX_ERR_NOT_FOUND
        return False


def layer_stream(vs, vps, idx, d, w, type_=b"tsdf", count=None, block_vps=None, trailing=b""):
    """voxblox io::SaveLayer's stream: varint32 message count, LayerProto, one BlockProto per block (unpacked
    voxel_data, colour 0)."""
    bs = F32(vs) * F32(vps)
    head = field(1, "d", float(vs)) + field(2, "v", int(vps)) + field(3, "L", type_)
    body = b""
    for b in range(len(idx)):
        bvps = block_vps if (block_vps is not None and b == 0) else vps
        blk = field(1, "v", int(bvps)) + field(2, "d", float(vs))
        blk += b"".join(field(3 + a, "d", float(F32(idx[b][a]) * bs)) for a in range(3)) + field(6, "v", 1)
        words = np.stack([np.asarray(d[b], F32).view(np.uint32), np.asarray(w[b], F32).view(np.uint32),
                          np.zeros(vps ** 3, np.uint32)], -1).reshape(-1)
        blk += b"".join(b"\x38" + varint(int(x)) for x in words)
        body += varint(len(blk)) + blk
    n = 1 + len(idx) if count is None else count
    return varint(n) + varint(len(head)) + head + body + trailing


def yaw_T(yaw, t=(0.0, 0.0, 0.0)):
    return np.array([np.cos(yaw / 2), 0, 0, np.sin(yaw / 2), *t], F32)


def poses_for(vs, vps):
    """Identity, a translation, a yaw and a random pose, scaled to the block size of (vs, vps)."""
    bs = float(F32(vs) * vps)
    rs = np.random.RandomState(int(vs * 1000) + vps)
    q = rs.normal(size=4); q /= np.linalg.norm(q)
    return {"identity": IDENTITY,
            "translation": np.array([1, 0, 0, 0, 2 * bs, -bs, 0.37 * bs], F32),
            "yaw": yaw_T(0.7, (0.3 * bs, 0.1 * bs, 0.0)),
            "random": np.array([*q, *rs.uniform(-bs, bs, 3)], F32)}


def oracle_layer(oracle, s):
    """The oracle Layer of a synth submap."""
    return oracle.Layer.from_blocks(s.voxel_size, s.vps, s.block_idx, s.distance, s.weight)


def compile_cpp_mirror(tmp_path, source):
    """Build the library and compile tests/cpp/<source> against its C-ABI and the C++ host mirror with
    plain g++ -> the executable."""
    from voxgraph_b200 import build
    build.build()
    exe = str(tmp_path / os.path.splitext(source)[0])
    lib_dir = os.path.join(ROOT, "voxgraph_b200")
    cmd = ["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"),
           "-I" + os.path.join(ROOT, "voxgraph_b200", "host"),
           os.path.join(ROOT, "tests", "cpp", source), "-o", exe,
           "-L" + lib_dir, "-lvoxgraph_b200", "-Wl,-rpath," + lib_dir]
    env = dict(os.environ); env.pop("CXX", None)
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    assert p.returncode == 0, p.stdout
    return exe


def build_oracle_harness(c_file, so_name, signatures):
    """Compile the C harness tests/<c_file> into a temporary directory (never into the tree; removed at
    exit), linked against oracle/libvg_oracle.so, whose layers it reads -> the loaded library, with the
    harness's {name: (restype, argtypes)} applied."""
    from oracle import oracle as o
    o.lib()   # builds and loads oracle/libvg_oracle.so first
    odir = os.path.join(ROOT, "oracle")
    tmp = tempfile.mkdtemp(prefix="vgx_%s_" % os.path.splitext(c_file)[0])
    atexit.register(shutil.rmtree, tmp, True)
    so = os.path.join(tmp, so_name)
    env = dict(os.environ)
    env.pop("CC", None)
    cmd = ["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-std=c11", "-Wall", "-Wextra",
           "-I" + odir, os.path.join(ROOT, "tests", c_file), "-o", so, "-L" + odir, "-lvg_oracle",
           "-Wl,-rpath," + odir, "-lm"]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    if p.returncode != 0:
        raise RuntimeError("building tests/%s failed:\n%s" % (c_file, p.stdout))
    L = C.CDLL(so)
    for name, (restype, argtypes) in signatures.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    return L


# The C headers that a ctypes table binds: the library's, the oracle's and the oracle harnesses' (which
# includes the oracle's).
LIBRARY_HEADER = os.path.join(ROOT, "include", "voxgraph_b200.h")
ORACLE_HEADER = os.path.join(ROOT, "oracle", "vg_oracle.h")
HARNESS_HEADER = os.path.join(ROOT, "tests", "oracle_harness.h")


def header_functions(header=LIBRARY_HEADER, prefix="vgx_"):
    """The names of the functions the header declares whose names start with prefix (a regular expression)."""
    hdr = re.sub(r"/\*.*?\*/", "", open(header).read(), flags=re.S)
    return set(re.findall(r"\b(%s\w+)\s*\(" % prefix, hdr))


def c_layout(tmp_path, structs, constants=(), header=LIBRARY_HEADER):
    """The C compiler's view of the header, from one gcc program: structs {typedef: [field names]} and
    constant names -> {typedef: sizeof, "typedef.field": offsetof, constant: value}."""
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % os.path.basename(header),
             'int main(void) {']
    for cname, fields in structs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname in fields:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    for name in constants:
        lines.append('printf("%s %%lld\\n", (long long)(%s));' % (name, name))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I" + os.path.dirname(header), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, stdout=subprocess.PIPE, text=True).stdout
    return {k: int(v) for k, v in (line.split() for line in out.splitlines())}


def check_struct_layouts(tmp_path, module, typedefs, header=LIBRARY_HEADER, constants=()):
    """Every ctypes.Structure the module defines has the size and field offsets of its typedef in the header
    (typedefs: {mirror name: typedef}, one entry per mirror), and every constant {name: value} the header's
    value."""
    mirrors = {n: v for n, v in vars(module).items()
               if isinstance(v, type) and issubclass(v, C.Structure) and v.__module__ == module.__name__}
    assert set(mirrors) == set(typedefs), "a ctypes struct without its header typedef, or a stale entry"
    structs = {typedefs[n]: ct for n, ct in mirrors.items()}
    out = c_layout(tmp_path, {c: [f for f, _ in ct._fields_] for c, ct in structs.items()}, constants, header)
    for cname, ct in structs.items():
        assert out[cname] == C.sizeof(ct), cname
        for fname, _ in ct._fields_:
            assert out["%s.%s" % (cname, fname)] == getattr(ct, fname).offset, (cname, fname)
    for name, value in dict(constants).items():
        assert out[name] == value, name
