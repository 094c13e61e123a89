"""Builds libsd_b200.so (hand-written sm_90a CUDA + the C ABI of include/sd_b200.h) in-tree with nvcc.

    python -m superviseddescent_b200.build            # incremental
    python -m superviseddescent_b200.build --force

The shared object lands in superviseddescent_b200/lib/ (git-ignored build product).  nvcc cross-compiles
for sm_90a (H100) without a GPU present.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
LIB = os.path.join(LIBDIR, "libsd_b200.so")

SOURCES = ["sd_api.cu", "sd_hog.cu", "sd_hog_dense.cu", "sd_hog_render.cu", "sd_hog_filters.cu", "sd_hog_detect.cu", "sd_hog_train.cu", "sd_hog_parts.cu", "sd_linalg.cu", "sd_gram_tc.cu", "sd_model.cu", "sd_comm.cu", "sd_rank.cu", "sd_cg.cu", "sd_train.cu", "sd_track.cu", "sd_face_chips.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo",
         "-Xcompiler", "-fPIC,-fvisibility=hidden", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    headers = [os.path.join(CSRC, "sd_internal.cuh"), os.path.join(CSRC, "sd_hog_common.cuh"), os.path.join(CSRC, "sd_warp.cuh"), os.path.join(ROOT, "include", "sd_b200.h")]
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append([NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        return cmd, r.returncode, r.stdout

    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        for cmd, rc, out in ex.map(run, jobs):
            if verbose or rc:
                sys.stderr.write(out)
            if rc:
                raise RuntimeError("nvcc failed: " + " ".join(cmd))
    if jobs or force or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart", "-ldl"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout)
            raise RuntimeError("link failed: " + " ".join(cmd))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
