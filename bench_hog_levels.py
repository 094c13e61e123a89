"""Per-level time of the landmark HOG kernel (sd_hog_batch) at the shape of bench.py's detect workload.

    python bench_hog_levels.py [--batch 4096] [--reps 20] [--warmup 3]

The frames and face boxes are bench.py's own, from the same seeds (4096 synthetic 640x480 frames generated on the GPU, one
box per frame); the landmarks are the mean shape aligned to each box, as the cascade's first level sees them.  For each of
the four cascade levels of the shipped model the projection runs with that level's HOG parameters (cell size, bins,
relative patch size).  One CUDA-event window per level after warm-up; the card's name, power limit and maximum SM clock
are read in the same run.  Prints one JSON line; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    import bench
    from bench_hog_dense import card
    from superviseddescent_b200 import _capi
    from superviseddescent_b200 import api as sd

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = sd.Context(0)
    model = sd.load_detection_model(bench.MODEL, ctx)
    B, L = args.batch, model.num_landmarks
    frames = bench.synth_frames_torch(B, 1234, dev)
    boxes = bench.synth_boxes(B, 1234)
    mean = model.get_mean()
    x0 = torch.from_numpy(np.stack([sd.align_mean(mean, b) for b in boxes])).to(dev)
    norm = sd.NormalisationC()
    _capi.lib().sd_model_normalisation(model._m, C.byref(norm))
    ib = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), bench.W_IMG, bench.H_IMG, frames.stride(1), frames.stride(0), B)

    levels = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for level in range(min(4, model.num_levels)):
        hp = model.hog_param(level)
        D = _capi.lib().sd_hog_feature_length(L, C.byref(hp))
        ld = (D + 3) // 4 * 4
        A = torch.empty((B, ld), dtype=torch.float32, device=dev)

        def hog():
            rc = _capi.lib().sd_hog_batch(ctx.h, C.byref(ib), None, _capi.ptr(x0), C.c_int64(2 * L), B, L, C.byref(norm),
                                          C.byref(hp), _capi.ptr(A), C.c_int64(ld))
            assert rc == 0, _capi.lib().sd_last_error(ctx.h)
        for _ in range(args.warmup):
            hog()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            hog()
        e1.record()
        torch.cuda.synchronize()
        levels.append({"level": level, "fs": hp.num_cells * hp.cell_size, "num_bins": hp.num_bins,
                       "ms_per_launch": e0.elapsed_time(e1) / args.reps})
        del A
    print(json.dumps({"metric": "hog_ms_per_level", "faces": B, "landmarks": L, "reps": args.reps, "levels": levels,
                      "total_ms": sum(v["ms_per_launch"] for v in levels), "card": card()}))


if __name__ == "__main__":
    main()
