"""Colour HOG pyramid (sd_hog_pyramid_images) against the grey one (sd_hog_pyramid), and colour against grey detection.

    python bench_hog_pyramid_images.py [--frames 64] [--reps 10] [--out FILE]

Workload: --frames B,G,R frames of 1280 x 720 per call, cell size 8, K = 9, UoCTTI, 21 levels at 2^(-l/5), l = 0 .. 20.  The
grey pyramid reads the frames' grey conversion (done once, outside the timing); the colour pyramid reads the interleaved
frames in place.  Per frame, with CUDA events: the grey and the colour pyramid alternated in one run; the colour pyramid with
bilinear orientations; and, from torch.profiler passes after the timed runs, one per pyramid because both resize with
hog_pyramid_resize_images_kernel, each pyramid's resize launches and HOG launches (hog_dense_kernel for the grey pyramid,
hog_images_kernel for the colour one).  Then vl_hog_detect end to end (host clock around a synchronised call, read-back included), grey against
colour, with Q = 2 (a 6 x 6-cell filter and its mirror).  The card's name, power limit and clock are read in the same run.
One JSON line per measurement; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

W, H, CS, K, VARIANT, LEVELS = 1280, 720, 8, 9, 1, 21


def card():
    """Name, power limit and max SM clock of GPU 0, read with nvidia-smi (None when it cannot be read)."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        name, power, clock = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return None


def bgr_frames(n, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    out = np.empty((n, H, W, 3), dtype=np.uint8)
    for c in range(3):
        base = 127.5 + 90 * np.sin(x / (19.0 + 4 * c) + np.cos(y / (29.0 + 3 * c))) * np.cos(y / (13.0 + 5 * c))
        for i in range(n):
            out[i, :, :, c] = np.clip(np.round(np.roll(base, 7 * i, axis=1) + rng.normal(0, 10, (H, W))), 0, 255)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_pyramid_images.py needs a CUDA device")
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import HogImageC, HogImagesC, ImageBatchC, ptr
    lib = _capi.lib()
    ctx = api.default_context()
    n = args.frames
    info = card()
    lines = []

    def emit(d):
        d["card"] = info
        print(json.dumps(d), flush=True)
        lines.append(d)

    scales = [2.0 ** (-l / 5) for l in range(LEVELS)]
    shapes = [api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)[1] for s in scales]
    per_frame = [d * h * w for d, h, w in shapes]
    offsets = [f * sum(per_frame) + sum(per_frame[:s]) for f in range(n) for s in range(LEVELS)]
    out = torch.empty(n * sum(per_frame), dtype=torch.float32, device="cuda")
    d_off = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    h_scales = (C.c_double * LEVELS)(*scales)

    bgr = torch.from_numpy(bgr_frames(n, 1)).cuda()
    grey = api.bgr2gray(bgr, ctx)
    gb = ImageBatchC(C.c_void_p(grey.data_ptr()), W, H, grey.stride(1), grey.stride(0), n)
    cb = HogImagesC()
    cb.d_data, cb.dtype, cb.channels, cb.count = bgr.data_ptr(), 0, 3, n
    cb.frame = HogImageC(W, H, 0, bgr.stride(1), bgr.stride(2), bgr.stride(3))
    cb.image_stride, cb.d_frames = bgr.stride(0), None

    def grey_call():
        api._check(ctx.h, lib.sd_hog_pyramid(ctx.h, C.byref(gb), h_scales, LEVELS, CS, K, VARIANT, ptr(out), ptr(d_off)))

    def colour_call(bil=0):
        api._check(ctx.h, lib.sd_hog_pyramid_images(ctx.h, C.byref(cb), h_scales, LEVELS, CS, K, VARIANT, bil, ptr(out), ptr(d_off)))

    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) * 1e3 / n           # microseconds per frame

    calls = {"grey": grey_call, "colour": colour_call, "colour_bilinear": lambda: colour_call(1)}
    for fn in calls.values():                                 # warm-up: module load, scratch growth
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, fn in calls.items():                           # alternated in one run
            times[k].append(timed(fn))
    for k, t in times.items():
        emit({"measure": f"pyramid_{k}", "us_per_frame_median": statistics.median(t), "us_per_frame_min": min(t),
              "us_per_frame_max": max(t), "reps": args.reps, "frames": n, "levels": LEVELS})
    emit({"measure": "colour_over_grey", "ratio_of_medians": statistics.median(times["colour"]) / statistics.median(times["grey"]),
          "bilinear_over_grey": statistics.median(times["colour_bilinear"]) / statistics.median(times["grey"])})

    # per-launch kernel times: a profiler pass of its own for each pyramid, whose resize launches share a kernel name
    from torch.profiler import ProfilerActivity, profile
    for route, call in (("grey", grey_call), ("colour", colour_call)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                call()
            torch.cuda.synchronize()
        per_kernel = {}
        for e in prof.key_averages():
            for name in ("hog_pyramid_resize_images_kernel", "hog_images_kernel", "hog_dense_kernel"):
                if name in e.key and e.device_type.name == "CUDA":
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    per_kernel[name] = per_kernel.get(name, 0.0) + t / 3 / n      # us per frame
        emit({"measure": f"pyramid_{route}_kernels_us_per_frame", **per_kernel})

    # vl_hog_detect end to end, grey against colour, Q = 2
    rng = np.random.default_rng(2)
    filt = torch.from_numpy(rng.normal(0, 0.1, (1, 3 * K + 4, 6, 6)).astype(np.float32)).cuda()
    filters = torch.cat([filt, api.vl_hog_flip(filt, K, VARIANT, ctx=ctx)])
    host_bgr = bgr

    def detect(mc):
        frames = host_bgr if mc else grey
        return api.vl_hog_detect(frames, scales, filters, CS, K, threshold=0.0, variant=VARIANT, max_detections=64, ctx=ctx,
                                 multichannel=mc)

    for mc in (False, True, False, True):
        detect(mc)
    dt = {False: [], True: []}
    for _ in range(args.reps):
        for mc in (False, True):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            detect(mc)
            torch.cuda.synchronize()
            dt[mc].append((time.perf_counter() - t0) * 1e6 / n)
    for mc in (False, True):
        emit({"measure": f"vl_hog_detect_{'colour' if mc else 'grey'}", "Q": 2, "levels": LEVELS, "us_per_frame_median": statistics.median(dt[mc]),
              "us_per_frame_min": min(dt[mc]), "us_per_frame_max": max(dt[mc]), "frames": n})
    if args.out:
        with open(args.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
