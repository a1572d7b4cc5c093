"""Builds agogo_b200/libagogo_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libagogo_b200.so")
OBJ = os.path.join(HERE, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]
# (file, extra flags).  -fmad=false: bit-exact PUCT / oracle-order fp32 arithmetic.
UNITS = [
    ("mcts.cu", ["-fmad=false"]),
    ("nn_fp32.cu", ["-fmad=false"]),
    ("tower_tc.cu", []),
    ("train_tc.cu", []),
    ("train.cu", []),
    ("engine.cu", []),
]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, ptxas_info=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "agogo_b200.h"))
    headers.append(os.path.abspath(__file__))
    objs = []
    for src, extra in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(o)
        if _stale(o, [s] + headers):
            cmd = [NVCC] + ARCH + COMMON + extra + (["-Xptxas", "-v"] if ptxas_info else []) + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd), flush=True)
            subprocess.check_call(cmd)
    if _stale(OUT, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", OUT] + objs + ["-lcudart", "-ldl", "-lpthread", "-ccbin", "/usr/bin/g++"]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(verbose=True, ptxas_info="-v" in sys.argv))
