"""TEST INFRASTRUCTURE: compile the kernels of madrl_b200/csrc with g++ against the fake
<cuda_runtime.h> of tests/emu/include into a CPU library with the product's C ABI
(tests/emu/_build/libmadrl_b200_emu_<tag>.so), loaded by tests/emu/driver.py."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "madrl_b200", "csrc")
OUT = os.path.join(HERE, "_build")
# every csrc/*.cu but exchange.cu, which needs the CUDA driver API
SOURCES = ["common.cu", "waterworld.cu", "pursuit.cu", "hostage.cu", "postproc.cu", "heuristics.cu", "baseline.cu"]
# The fixed reduction grids of postproc.cu and baseline.cu (on the GPU: 528 moment blocks of 256 threads, 64, 32
# and 48 row slices), narrowed so that a launch does not create a hundred thousand fibers.  Tests that put their
# sizes at the grids' edges read them here.
GRID = {"MADRL_MOM_BLOCKS": 6, "MADRL_RM_SLICES": 3, "MADRL_TB_SLICES": 3, "MADRL_LFB_SLICES": 3}
# the shared arrays of these two files are block-static, not `extern`
PER_FILE_FLAGS = {f: ["-D__shared__=static"] + ["-D%s=%d" % kv for kv in GRID.items()]
                  for f in ("postproc.cu", "baseline.cu")}
CXXFLAGS = ["-std=c++17", "-O1", "-g", "-fPIC", "-Wno-unknown-pragmas", "-Wno-attributes", "-x", "c++",
            "-I", os.path.join(HERE, "include")]


def _deps():
    out = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    out += [os.path.join(HERE, "include", "cuda_runtime.h"), os.path.join(HERE, "emu_runtime.cpp"),
            os.path.join(ROOT, "include", "madrl_b200.h"), os.path.abspath(__file__)]
    return out


def build(defines=(), force=False):
    """Returns the path of the emulator library built with the given -D flags."""
    tag = hashlib.sha1(" ".join(sorted(defines)).encode()).hexdigest()[:10] if defines else "default"
    lib = os.path.join(OUT, "libmadrl_b200_emu_%s.so" % tag)
    if not force and os.path.exists(lib) and all(os.path.getmtime(d) <= os.path.getmtime(lib) for d in _deps()):
        return lib
    objdir = os.path.join(OUT, "obj_" + tag)
    os.makedirs(objdir, exist_ok=True)
    cxx = os.environ.get("CXX", "g++")

    def one(src):
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        cmd = [cxx] + CXXFLAGS + list(defines) + PER_FILE_FLAGS.get(os.path.basename(src), []) + ["-c", "-o", obj, src]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if res.returncode:
            sys.stderr.write(res.stdout)
            raise RuntimeError("g++ failed: " + " ".join(cmd))
        return obj

    srcs = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.join(HERE, "emu_runtime.cpp")]
    with ThreadPoolExecutor(max_workers=len(srcs)) as pool:
        objs = list(pool.map(one, srcs))
    tmp = lib + ".%d.tmp" % os.getpid()
    subprocess.check_call([cxx, "-shared", "-o", tmp] + objs)
    os.replace(tmp, lib)
    return lib


if __name__ == "__main__":
    print(build([a for a in sys.argv[1:] if a.startswith("-D")], force="--force" in sys.argv))
