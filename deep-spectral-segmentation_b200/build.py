"""In-tree build of libdss_b200.so with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python deep-spectral-segmentation_b200/build.py [--force]

The shared object lands next to this file (git-ignored); object files and the compiler log go to build/.
"""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "libdss_b200.so"
SOURCES = ["api.cu", "gemm.cu", "vit_kernels.cu", "attention.cu", "vit.cu", "affinity.cu", "eigsh.cu", "knn.cu", "segment.cu",
           "cluster.cu", "crf.cu", "localize.cu", "segeval.cu", "resize.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "-DDSS_BUILD", "-Xptxas", "-v", *os.environ.get("DSS_EXTRA_NVCC_FLAGS", "").split()]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (Path(cand).is_file() or cand == "nvcc"):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not LIB.is_file():
        return True
    t = LIB.stat().st_mtime
    deps = [CSRC / s for s in SOURCES] + [CSRC / "common.cuh", CSRC / "gemm_pipeline.cuh", CSRC / "kmeans_common.cuh", HERE.parent / "include" / "dss_b200.h", Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    objdir = HERE / "build"
    objdir.mkdir(exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for s in SOURCES:
        o = objdir / (s[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / s), "-o", str(o)]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(o))
    log = []
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {s}\n{out}")
        failed |= p.returncode != 0
    (objdir / "build.log").write_text("\n".join(log))
    if failed or verbose:
        print("\n".join(log))
    if failed:
        raise RuntimeError("nvcc failed, see above")
    cmd = [nvcc, *NVCC_FLAGS[:2], "-shared", "-o", str(LIB), *objs, "-cudart", "static"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
