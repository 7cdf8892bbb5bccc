"""In-tree build of libsvsdf_b200.so for the H100 (sm_90a only; nvcc cross-compiles without a GPU).

    python -m implicit_svsdf_planner_b200.build [--force] [--verbose]

Outputs: implicit_svsdf_planner_b200/lib/libsvsdf_b200.so (+ object files under lib/obj/), both git-ignored.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
SO = os.path.join(LIBDIR, "libsvsdf_b200.so")

NVCC = os.environ.get("SVSDF_NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-ccbin", "/usr/bin/g++"]
COMMON += os.environ.get("SVSDF_EXTRA_NVCC_FLAGS", "").split()  # experiments, e.g. -DSVSDF_OUTER_MIN_CTAS=4

UNITS = [
    # (source, object, extra flags)
    ("svsdf_kernels_fast.cu", "svsdf_kernels_fast.o", []),
    ("svsdf_kernels_strict.cu", "svsdf_kernels_strict.o", ["-fmad=false"]),
    ("svsdf_extract.cu", "svsdf_extract.o", ["-fmad=false"]),  # cell centres must round like the host formula
    ("svsdf_frontend.cu", "svsdf_frontend.o", ["-fmad=false"]),  # shape kernels: same rounding as the strict functors
    # host threads for the batch A* bookkeeping; no a*b+c contraction in the float winding-number builder (host/fwn_bvh.hpp)
    ("svsdf_runtime.cpp", "svsdf_runtime.o", ["-Xcompiler", "-fopenmp", "-Xcompiler", "-ffp-contract=off"]),
]
HEADERS = [
    "svsdf_kernels.cuh",
    "svsdf_shapes.cuh",
    "svsdf_sincos.cuh",
    "svsdf_types.h",
    "svsdf_launch.h",
    "host/minco.hpp",
    "host/lbfgs.hpp",
    "host/astar.hpp",
    "host/astar_flat.hpp",
    "host/fwn_bvh.hpp",
    "host/mid_end.hpp",
    "../../include/svsdf.h",
]


def _mtime(p):
    return os.path.getmtime(p) if os.path.exists(p) else 0.0


def _cmd(unit):
    src, obj, extra = unit
    return [NVCC, *ARCH, *COMMON, *extra, "-c", os.path.join(CSRC, src), "-o", os.path.join(OBJDIR, obj)]


def _compile(unit, verbose):
    src, obj, extra = unit
    cmd = _cmd(unit)
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    with open(os.path.join(OBJDIR, obj + ".cmd"), "w") as fh:  # rebuild when the flags change, not only the sources
        fh.write(" ".join(_cmd(unit)))
    return r.stderr if verbose else ""


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJDIR, exist_ok=True)
    newest_hdr = max(_mtime(os.path.join(CSRC, h)) for h in HEADERS)
    todo = []
    for u in UNITS:
        src_t = max(_mtime(os.path.join(CSRC, u[0])), newest_hdr)
        stamp = os.path.join(OBJDIR, u[1] + ".cmd")
        same_cmd = os.path.exists(stamp) and open(stamp).read() == " ".join(_cmd(u))
        if force or not same_cmd or _mtime(os.path.join(OBJDIR, u[1])) < src_t:
            todo.append(u)
    if todo:
        with cf.ThreadPoolExecutor(max_workers=len(todo)) as ex:
            for out in ex.map(lambda u: _compile(u, verbose), todo):
                if out:
                    print(out)
    objs = [os.path.join(OBJDIR, u[1]) for u in UNITS]
    if todo or not os.path.exists(SO) or _mtime(SO) < max(_mtime(o) for o in objs):
        cmd = [NVCC, *ARCH, "-shared", "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fopenmp", "-o", SO, *objs, "-lgomp"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
