"""Build libpvn3d_b200.so (hand-written sm_90a kernels + the C ABI of include/pvn3d_b200.h).

Plain `nvcc -shared`: the library links only against the CUDA runtime -- no torch, no ATen -- so
the boundary stays a C ABI (plain pointers and sizes).  The .so is written IN-TREE next to this
file and git-ignored.

    python -m pvn3d_b200.build            # incremental
    python -m pvn3d_b200.build --force
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libpvn3d_b200.so")
SOURCES = ["runtime.cu", "fps.cu", "pn2_ops.cu", "query_group.cu", "meanshift.cu", "poses.cu", "mlp_tc.cu", "metrics.cu",
           "icp.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-I", os.path.join(ROOT, "include"),
    "-I", CSRC,
]


def _newer(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps if os.path.exists(d))


def _compile(src: str, verbose: bool) -> str:
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    deps = [os.path.join(CSRC, src), os.path.join(CSRC, "common.cuh"),
            os.path.join(ROOT, "include", "pvn3d_b200.h"), os.path.abspath(__file__)]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    if _newer(obj, deps):
        return obj
    cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose:
        sys.stderr.write(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every .cu for sm_90a and link the shared library.  Returns its path."""
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            return LIB  # machine without a toolkit: use the library built beforehand
        raise RuntimeError("nvcc not found and no prebuilt libpvn3d_b200.so in tree")
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if not _newer(LIB, objs):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a",
               "-Xcompiler", "-fPIC", "-lcudart_static", "-lrt", "-lpthread", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
