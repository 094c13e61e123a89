"""HOG pyramid and filter scores (sd_hog_pyramid, sd_hog_correlate): the two steps of a sliding-window detector on the GPU.

    python bench_hog_filters.py [--frames 64] [--reps 10] [--out FILE]

Workload: 1280x720 grey frames, --frames per call, cell size 8, K = 9, UoCTTI; scales 2^(-l/5), l = 0, 1, ... while the level
holds at least a 6 x 6-cell filter; a 6 x 6-cell filter bank at pad 0 with Q = 1, 2 (a filter and its mirror) and 32.  It
reports the CUDA-event time of the pyramid and of the scoring separately, frames/s, the library's launches per call
(sd_launch_count), and for the scoring the algorithmic flops sum(outputs) * Q * 2 * dd * fh * fw and bytes (maps read once,
filters, scores written) as shares of 67 TFLOP/s (H100 SXM FP32, dense) and 3.35 TB/s (HBM3), naming the bound that applies.
As a comparison only, torch.nn.functional.conv2d in fp32 with TF32 off scores the same maps, one call per level (the frames of
a level stacked into one batch beforehand).  The card's name and power limit are read in the same run.  One JSON line per
setting; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
FP32_FLOPS_PER_S = 67e12
W, H, CS, K, VARIANT, FH, FW = 1280, 720, 8, 9, 1, 6, 6
BANKS = [1, 2, 32]


def card():
    """Name, power limit and max SM clock of GPU 0, read with nvidia-smi (None when it cannot be read)."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        name, power, clock = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return None


def frames_for(n, w, h, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = 127.5 + 90 * np.sin(x / 23.0 + np.cos(y / 31.0)) * np.cos(y / 17.0)
    out = np.empty((n, h, w), dtype=np.uint8)
    for i in range(n):
        out[i] = np.clip(np.round(np.roll(base, 7 * i, axis=1) + rng.normal(0, 10, (h, w))), 0, 255)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_filters.py needs a CUDA device")
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import HogGridC, HogGridsC, ImageBatchC, ptr
    lib = _capi.lib()
    ctx = api.default_context()
    n = args.frames
    info = card()

    scales, l = [], 0
    while True:
        s = 2.0 ** (-l / 5)
        (_, _), (dd, hh, hw) = api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)
        if hh < FH or hw < FW:
            break
        scales.append(s)
        l += 1
    shapes = [api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)[1] for s in scales]
    per_frame = [d * h * w for d, h, w in shapes]
    offsets = [f * sum(per_frame) + sum(per_frame[:i]) for f in range(n) for i in range(len(scales))]
    frames = torch.from_numpy(frames_for(n, W, H, 1)).cuda()
    ib = ImageBatchC(C.c_void_p(frames.data_ptr()), W, H, W, W * H, n)
    out = torch.empty(n * sum(per_frame), dtype=torch.float32, device="cuda")
    d_off = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    h_scales = (C.c_double * len(scales))(*scales)

    def pyramid():
        api._check(ctx.h, lib.sd_hog_pyramid(ctx.h, C.byref(ib), h_scales, len(scales), CS, K, VARIANT, ptr(out), ptr(d_off)))

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        l0 = lib.sd_launch_count(ctx.h)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps * 1e-3, (lib.sd_launch_count(ctx.h) - l0) / reps

    t_pyr, launches_pyr = timed(pyramid, args.reps)
    cells = sum(h * w for _, h, w in shapes)
    rec = {"setting": "pyramid", "frames": n, "levels": len(scales), "cells_per_frame": cells, "pyramid_s": t_pyr,
           "us_per_frame": t_pyr / n * 1e6, "frames_per_s": n / t_pyr, "launches_per_call": launches_pyr, "card": info}
    print(json.dumps(rec), flush=True)
    results = [rec]

    # the maps: every level of every frame, read in place from the pyramid's buffer
    descs = []
    for f in range(n):
        for i, (d, h, w) in enumerate(shapes):
            oh, ow = h - FH + 1, w - FW + 1
            descs.append((w, h, offsets[f * len(scales) + i], oh, ow))
    map_bytes = 4 * n * sum(per_frame)
    stacked = [torch.stack([out[offsets[f * len(scales) + i]:offsets[f * len(scales) + i] + per_frame[i]].view(shapes[i])
                            for f in range(n)]) for i in range(len(scales))]
    rng = np.random.default_rng(2)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for Q in BANKS:
        filt = torch.from_numpy(rng.normal(0, 1, (Q, 3 * K + 4, FH, FW)).astype(np.float32)).cuda()
        table, pos = [], 0
        for w, h, off, oh, ow in descs:
            table.append(HogGridC(w, h, off, pos))
            pos += Q * oh * ow
        outputs = sum(oh * ow for _, _, _, oh, ow in descs)
        d_table = torch.from_numpy(np.frombuffer(bytes((HogGridC * len(table))(*table)), dtype=np.uint8).copy()).cuda()
        g = HogGridsC()
        g.d_features, g.count, g.width, g.height, g.d_grids = out.data_ptr(), len(table), 0, 0, d_table.data_ptr()
        scores = torch.empty(pos, dtype=torch.float32, device="cuda")

        def score():
            api._check(ctx.h, lib.sd_hog_correlate(ctx.h, C.byref(g), K, VARIANT, ptr(filt), Q, FW, FH, None, 0, 0, ptr(scores)))

        t, launches = timed(score, args.reps)
        flops = outputs * Q * 2 * (3 * K + 4) * FH * FW
        nbytes = map_bytes + 4 * filt.numel() + 4 * outputs * Q
        t_flop, t_byte = flops / FP32_FLOPS_PER_S, nbytes / HBM_BYTES_PER_S
        bound = "fp32" if t_flop >= t_byte else "hbm"

        def conv():
            for m in stacked:
                torch.nn.functional.conv2d(m, filt)

        t_conv, _ = timed(conv, args.reps)
        rec = {"setting": f"score Q={Q}", "frames": n, "grids": len(table), "outputs_per_frame": outputs // n, "score_s": t,
               "us_per_frame": t / n * 1e6, "frames_per_s": n / t, "launches_per_call": launches,
               "gflop_per_frame": flops / n / 1e9, "map_mb_per_frame": map_bytes / n / 1e6,
               "tflop_per_s": flops / t / 1e12, "share_fp32": t_flop / t, "gb_per_s": nbytes / t / 1e9, "share_hbm": t_byte / t,
               "bound": bound, "share_of_bound": max(t_flop, t_byte) / t,
               "comparison_only_torch_conv2d_fp32_s": t_conv, "comparison_only_us_per_frame": t_conv / n * 1e6, "card": info}
        print(json.dumps(rec), flush=True)
        results.append(rec)
    if args.out:
        with open(args.out, "w") as f:
            for r in results:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
