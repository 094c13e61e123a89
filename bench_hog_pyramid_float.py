"""Float HOG pyramid (sd_hog_pyramid_float) against the 8-bit colour one (sd_hog_pyramid_images) on the same frames.

    python bench_hog_pyramid_float.py [--frames 64] [--reps 10] [--out FILE]

Workload: --frames frames of 1280 x 720 per call with four channels, B, G, R and grey, cell size 8, K = 9, UoCTTI, 21 levels at
2^(-l/5), l = 0 .. 20: the workload of bench_hog_pyramid_images.py with the grey channel added, so both pyramids vote over the
same four channels.  The 8-bit pyramid reads uint8 frames and the float pyramid float32 frames holding the same values, both
interleaved and in place.  Per frame, with CUDA events: the two pyramids alternated in one run; then, from a torch.profiler
pass of each route on its own after the timed runs, its resize (hog_pyramid_resize_images_kernel) and HOG (hog_images_kernel)
launches, and the bytes the resize reads and writes per frame over its time.  The card's name, power limit and clock are read
in the same run.  One JSON line per measurement; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_hog_pyramid_images import H, W, CS, K, LEVELS, VARIANT, bgr_frames, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_pyramid_float.py needs a CUDA device")
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import HogImageC, HogImagesC, ptr
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
    u8 = torch.cat([bgr, api.bgr2gray(bgr, ctx)[..., None]], dim=3).contiguous()       # B, G, R, grey
    f32 = u8.float()
    del bgr

    def batch(t, dtype):
        b = HogImagesC()
        b.d_data, b.dtype, b.channels, b.count = t.data_ptr(), dtype, 4, n
        b.frame = HogImageC(W, H, 0, t.stride(1), t.stride(2), t.stride(3))
        b.image_stride, b.d_frames = t.stride(0), None
        return b

    ub, fb = batch(u8, 0), batch(f32, 1)

    def u8_call():
        api._check(ctx.h, lib.sd_hog_pyramid_images(ctx.h, C.byref(ub), h_scales, LEVELS, CS, K, VARIANT, 0, ptr(out), ptr(d_off)))

    def float_call():
        api._check(ctx.h, lib.sd_hog_pyramid_float(ctx.h, C.byref(fb), h_scales, LEVELS, CS, K, VARIANT, 0, ptr(out), ptr(d_off)))

    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        start.record()
        fn()
        stop.record()
        stop.synchronize()
        return start.elapsed_time(stop) * 1e3 / n           # microseconds per frame

    calls = {"u8": u8_call, "float": float_call}
    for fn in calls.values():                                 # warm-up: module load, scratch growth
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    for _ in range(args.reps):
        for k, fn in calls.items():                           # alternated in one run
            times[k].append(timed(fn))
    for k, t in times.items():
        emit({"measure": f"pyramid_{k}_4ch", "us_per_frame_median": statistics.median(t), "us_per_frame_min": min(t),
              "us_per_frame_max": max(t), "reps": args.reps, "frames": n, "levels": LEVELS})
    emit({"measure": "float_over_u8", "ratio_of_medians": statistics.median(times["float"]) / statistics.median(times["u8"])})

    # per-launch kernel times, one profiler pass per route
    from torch.profiler import ProfilerActivity, profile
    level_px = sum(w * h for w, h in (api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)[0] for s in scales) if (w, h) != (W, H))
    for k, fn in calls.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
        per_kernel = {}
        for e in prof.key_averages():
            for name in ("hog_pyramid_resize_images_kernel", "hog_images_kernel"):
                if name in e.key and e.device_type.name == "CUDA":
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    per_kernel[name] = per_kernel.get(name, 0.0) + t / 3 / n          # us per frame
        # the resize writes every level once (4 channels, the copied scale-1 level included) and reads the frame at least once
        es = 4 if k == "float" else 1
        bytes_per_frame = es * 4 * (level_px + W * H) + es * 4 * W * H
        rs = per_kernel.get("hog_pyramid_resize_images_kernel", 0.0)
        emit({"measure": f"pyramid_{k}_kernels_us_per_frame", **per_kernel,
              "resize_min_bytes_per_frame": bytes_per_frame, "resize_GBps": bytes_per_frame / rs / 1e3 if rs else None})
    if args.out:
        with open(args.out, "w") as f:
            for d in lines:
                f.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
