"""In-tree build of libvoxgraph_b200.so (hand-written CUDA for sm_90a + the C-ABI)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
LIB = os.path.join(HERE, "libvoxgraph_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-I" + INCLUDE, "-I" + CSRC]
# (source, extra flags). -fmad=false: the reference's float expressions are restated
# operation by operation (see registration.cuh); graph.cu and solve.cu are double-precision pose-graph code.
SOURCES = [
    ("submap.cu", ["-fmad=false"]),
    ("registration.cu", ["-fmad=false"]),
    ("tsdf.cu", ["-fmad=false"]),
    ("extract.cu", ["-fmad=false"]),
    ("overlap.cu", ["-fmad=false"]),
    ("esdf.cu", ["-fmad=false"]),
    ("graph.cu", []),
    ("solve.cu", []),
    ("p2p.cu", []),
    ("nccl_dyn.cpp", []),
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src, extra in SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(objdir, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc] + ARCH + COMMON + extra + ["-c", path, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out))
        elif verbose:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("CUDA build failed")
    cmd = [nvcc] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart", "-ldl"]
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
