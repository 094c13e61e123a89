"""The rest of VLFeat's HOG object API on the GPU: render, relayout, column-major frames and the hog.h drop-in's per-call latency.

    python bench_vl_hog_api.py [--reps 20] [--warmup 3] [--calls 200]

In one run, with the card's name and power limit read alongside:
  render     sd_hog_render of 64 grids of 240 x 135 cells at K = 9 (UoCTTI): kernel time from CUDA events, and GB/s of the bytes
             it must move (the 3K planes it reads + the image read and written) against the H100 SXM's 3.35 TB/s;
  relayout   sd_hog_relayout of the same features, flip and transpose: GB/s of one read and one write of every plane;
  colmajor   sd_hog_dense_images frames/s on 64 f32 1280 x 720 frames, cell size 8, K = 9: row-major frames, against the same
             frames column-major (read through swapped strides, then the planes transposed by sd_hog_relayout), as the hog.h
             drop-in's transposed mode runs them;
  drop-in    us per vl_hog_put_image + vl_hog_extract through superviseddescent_b200/include/rcr/hog.h (a small C++ library
             compiled into a temporary directory at run time), next to the reference's hog.c (oracle/_ref) in the same process,
             for a 55 x 55 patch (cell size 11, K = 4) and a 1280 x 720 frame (cell size 8, K = 9).
One JSON line per row; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_hog_dense import card  # noqa: E402

PEAK_BW = 3.35e12
SHELL_SRC = r'''
#include "rcr/hog.h"
extern "C" double shell_put_extract(const float* img, int w, int h, int cs, int K, int calls, float* out)
{
    VlHog* hog = vl_hog_new(VlHogVariantUoctti, K, VL_FALSE);
    vl_hog_put_image(hog, img, w, h, 1, cs);
    vl_hog_extract(hog, out);                                   // warm-up: buffers sized, context created
    auto t0 = std::chrono::steady_clock::now();
    for (int i = 0; i < calls; ++i) { vl_hog_put_image(hog, img, w, h, 1, cs); vl_hog_extract(hog, out); }
    const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    vl_hog_delete(hog);
    return s;
}
'''


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def grids(t, count, w, h):
    from superviseddescent_b200._capi import HogGridsC
    g = HogGridsC()
    g.d_features, g.count, g.width, g.height, g.d_grids = t.data_ptr(), count, w, h, None
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--calls", type=int, default=200, help="drop-in calls per size")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vl_hog_api.py measures the GPU: no CUDA device")
    from superviseddescent_b200 import _capi, api as sd
    lib, ctx = _capi.lib(), sd.default_context()
    info = card()
    print(json.dumps({"card": info}))

    def check(rc):
        if rc:
            raise RuntimeError(lib.sd_last_error(ctx.h).decode())

    # render and relayout: 64 grids of 240 x 135 cells, K = 9, UoCTTI
    B, K, w, h = 64, 9, 240, 135
    dd = 3 * K + 4
    feats = torch.randn(B, dd, h, w, device="cuda")
    g = grids(feats, B, w, h)
    image = torch.zeros(B, h * 21, w * 21, device="cuda")
    t = timed(lambda: check(lib.sd_hog_render(ctx.h, C.byref(g), K, 1, 0, _capi.ptr(image))), args.reps, args.warmup)
    nbytes = B * 3 * K * w * h * 4 + 2 * image.numel() * 4
    print(json.dumps({"row": "render", "grids": B, "cells": [w, h], "K": K, "ms": t * 1e3, "GB_per_s": nbytes / t / 1e9,
                      "share_of_3.35TB_per_s": nbytes / t / PEAK_BW}))
    del image
    out = torch.empty_like(feats)
    for name, flip, tr in [("flip", 1, 0), ("transpose", 0, 1), ("flip+transpose", 1, 1)]:
        t = timed(lambda: check(lib.sd_hog_relayout(ctx.h, C.byref(g), K, 1, flip, tr, _capi.ptr(out))), args.reps, args.warmup)
        nbytes = 2 * feats.numel() * 4
        print(json.dumps({"row": "relayout", "op": name, "grids": B, "cells": [w, h], "dd": dd, "us": t * 1e6,
                          "GB_per_s": nbytes / t / 1e9, "share_of_3.35TB_per_s": nbytes / t / PEAK_BW}))
    del feats, out

    # column-major frames: swapped strides + relayout, against row-major
    n, W, H, cs = 64, 1280, 720, 8
    rows = torch.rand(n, H, W, device="cuda") * 255
    cols = rows.transpose(1, 2).contiguous().transpose(1, 2)            # same pixels, column-major in memory
    hw, hh = (W + cs // 2) // cs, (H + cs // 2) // cs
    planes = torch.empty(n, dd, hh, hw, device="cuda")
    gp = grids(planes, n, hw, hh)
    res = {}
    for name, frames in [("row-major", rows), ("column-major", cols)]:
        def run():
            f = sd.vl_hog(frames, cs, K, 1)
            if name == "column-major":
                gp.d_features = f.data_ptr()
                check(lib.sd_hog_relayout(ctx.h, C.byref(gp), K, 1, 0, 1, _capi.ptr(planes)))
        t = timed(run, args.reps, args.warmup)
        res[name] = n / t
        print(json.dumps({"row": "colmajor", "layout": name, "frames": n, "size": [W, H], "cs": cs, "K": K, "frames_per_s": n / t}))
    print(json.dumps({"row": "colmajor", "column_over_row": res["column-major"] / res["row-major"]}))
    del rows, cols, planes

    # the drop-in's latency per put_image + extract, next to hog.c
    tmp = tempfile.mkdtemp()
    so = os.path.join(tmp, "libshell_bench.so")
    src = os.path.join(tmp, "shell_bench.cpp")
    with open(src, "w") as f:
        f.write("#include <chrono>\n" + SHELL_SRC)
    libdir = os.path.join(ROOT, "superviseddescent_b200", "lib")
    subprocess.run(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include"), "-I",
                    os.path.join(ROOT, "superviseddescent_b200", "include"), src, "-L", libdir, "-lsd_b200", f"-Wl,-rpath,{libdir}",
                    "-o", so], check=True)
    shell = C.CDLL(so)
    shell.shell_put_extract.restype = C.c_double
    shell.shell_put_extract.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    try:
        from oracle import vl_hog_api_ref
        ref = vl_hog_api_ref if vl_hog_api_ref.available() else None
    except Exception:
        ref = None
    rng = np.random.default_rng(0)
    for (pw, ph, cs, k) in [(55, 55, 11, 4), (1280, 720, 8, 9)]:
        img = (rng.random((ph, pw)) * 255).astype(np.float32)
        d = 3 * k + 4
        buf = np.empty(d * ((ph + cs // 2) // cs) * ((pw + cs // 2) // cs), np.float32)
        calls = args.calls if pw < 256 else max(args.calls // 10, 5)
        s = shell.shell_put_extract(img.ctypes.data, pw, ph, cs, k, calls, buf.ctypes.data)
        row = {"row": "drop-in", "size": [pw, ph], "cs": cs, "K": k, "calls": calls, "shell_us_per_call": s / calls * 1e6}
        if ref is not None:
            hog = ref.Hog(1, k)
            hog.put_image(img, cs)
            t0 = time.perf_counter()
            for _ in range(calls):
                hog.put_image(img, cs)
            row["hog_c_us_per_call"] = (time.perf_counter() - t0) / calls * 1e6
        else:
            row["hog_c_us_per_call"] = "not measured (oracle/_ref absent)"
        print(json.dumps(row))


if __name__ == "__main__":
    main()
