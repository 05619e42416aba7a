"""Build libdampr_b200.so in-tree with nvcc for sm_90a (H100; no JIT cache, the .so travels with the repo)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdampr_b200.so")
SOURCES = ["ctx.cu", "text.cu", "text2.cu", "kv.cu", "merge.cu", "ops.cu", "comm.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    """Compile every .cu into build/*.o and link the shared library. Returns the library path."""
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    deps = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "leaf.cuh"), os.path.join(HERE, "..", "include", "dampr_b200.h")]
    objs = []
    relink = force or not os.path.exists(LIB)
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(s, o) or any(_newer(d, o) for d in deps):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), file=sys.stderr)
            subprocess.check_call(cmd)
            relink = True
    if relink:
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ARCH + ["-ldl"]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
