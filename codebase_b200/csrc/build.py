"""Builds codebase_b200/csrc/libmarlb200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libmarlb200.so")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + [
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "--expt-relaxed-constexpr",
]


def sources():
    return sorted(glob.glob(os.path.join(HERE, "*.cu")))


def needs_build() -> bool:
    if not os.path.exists(SO):
        return True
    deps = sources() + glob.glob(os.path.join(HERE, "*.cuh")) + [os.path.join(HERE, "..", "..", "include", "marl_b200.h")]
    return any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps)


def build(force: bool = False, verbose: bool = False, out: str | None = None, defines: list[str] | None = None) -> str:
    """`out` / `defines`: a second, profiling build next to the product library (e.g. -DMARL_TC_TIMESTAMPS -> libmarlb200_ts.so, loaded with
    MARL_B200_SO=<path>); the product library is always built without extra defines unless MARL_NVCC_DEFINES says otherwise."""
    target = out or SO
    if out is None and not force and not needs_build():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = (defines if defines is not None else os.environ.get("MARL_NVCC_DEFINES", "").split())
    srcs = sources()
    if os.environ.get("MARL_PARALLEL_BUILD", "1") == "1":   # one nvcc per translation unit, in parallel, then link
        import concurrent.futures as cf
        objdir = os.path.join(HERE, "build", os.path.basename(target))
        os.makedirs(objdir, exist_ok=True)
        flags = [f for f in NVCC_FLAGS if f != "-shared"]
        def cc(src):
            obj = os.path.join(objdir, os.path.basename(src) + ".o")
            subprocess.check_call([nvcc] + flags + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj], cwd=HERE)
            return obj
        with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
            objs = list(ex.map(cc, srcs))
        subprocess.check_call([nvcc] + GENCODE + ["-shared", "-o", target] + objs, cwd=HERE)
    else:
        subprocess.check_call([nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", target] + srcs, cwd=HERE)
    return target


if __name__ == "__main__":
    if "--timestamps" in sys.argv:
        print(build(force=True, out=os.path.join(HERE, "libmarlb200_ts.so"), defines=["-DMARL_TC_TIMESTAMPS"]))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
