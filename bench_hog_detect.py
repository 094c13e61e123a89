"""Detections from HOG filter scores (sd_hog_detections): the last step of a sliding-window detector on the GPU.

    python bench_hog_detect.py [--frames 64] [--reps 10] [--out FILE]

Workload: bench_hog_filters.py's -- 1280x720 grey frames, --frames per call, cell size 8, K = 9, UoCTTI, scales 2^(-l/5) while a
level holds the 6 x 6-cell filter, banks of Q = 1, 2 and 32 random filters at pad 0.  Per bank it times, with CUDA events:
the pyramid and the scoring (the cost the detection step is compared with), and sd_hog_detections alone at three thresholds taken
from the score quantiles so that a frame has about 50, about 2,000, and more than max_candidates (4096) candidates, with
max_detections 256 and overlap 0.5.  It reports the detection step's share of pyramid + scores.  End to end, vl_hog_detect on the
device frames in frames/s at Q = 1 and 2, and one frame at Q = 2 (the video case), timed on the host clock around calls that end
in a download.  As a comparison only: torch thresholding + topk (max_candidates per frame) + torchvision.ops.batched_nms on the
same scores, with the boxes precomputed outside the timing; null when torchvision's CUDA ops do not load.  The card's name and
power limit are read in the same run.  One JSON line per setting; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_hog_filters import CS, FH, FW, H, K, VARIANT, W, card, frames_for  # noqa: E402

BANKS = [1, 2, 32]
MAX_C, MAX_DET, OVERLAP = 4096, 256, 0.5
TARGETS = [("about 50", 50), ("about 2000", 2000), ("over max_candidates", 3 * MAX_C)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_detect.py needs a CUDA device")
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import HogGridC, HogGridsC, HogScoreMapC, ImageBatchC, ptr
    lib = _capi.lib()
    ctx = api.default_context()
    n = args.frames
    info = card()
    try:
        import torchvision
        torchvision.ops.batched_nms(torch.zeros((1, 4), device="cuda"), torch.zeros(1, device="cuda"),
                                    torch.zeros(1, dtype=torch.int64, device="cuda"), 0.5)
        tv = torchvision
    except Exception:
        tv = None

    scales, l = [], 0
    while True:
        s = 2.0 ** (-l / 5)
        (_, _), (_, hh, hw) = api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)
        if hh < FH or hw < FW:
            break
        scales.append(s)
        l += 1
    levels = [api.hog_pyramid_shape(W, H, s, CS, K, VARIANT) for s in scales]
    per_frame = [d * h * w for _, (d, h, w) in levels]
    offsets = [f * sum(per_frame) + sum(per_frame[:i]) for f in range(n) for i in range(len(scales))]
    frames = torch.from_numpy(frames_for(n, W, H, 1)).cuda()
    ib = ImageBatchC(C.c_void_p(frames.data_ptr()), W, H, W, W * H, n)
    feats = torch.empty(n * sum(per_frame), dtype=torch.float32, device="cuda")
    d_off = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    h_scales = (C.c_double * len(scales))(*scales)

    def pyramid():
        api._check(ctx.h, lib.sd_hog_pyramid(ctx.h, C.byref(ib), h_scales, len(scales), CS, K, VARIANT, ptr(feats), ptr(d_off)))

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps * 1e-3

    t_pyr = timed(pyramid, args.reps)
    results = []
    rng = np.random.default_rng(2)
    for Q in BANKS:
        filt = torch.from_numpy(rng.normal(0, 1, (Q, 3 * K + 4, FH, FW)).astype(np.float32)).cuda()
        grids, maps, pos = [], [], 0
        for f in range(n):
            for i, ((lw, lh), (_, h, w)) in enumerate(levels):
                oh, ow = h - FH + 1, w - FW + 1
                grids.append(HogGridC(w, h, offsets[f * len(scales) + i], pos))
                maps.append(HogScoreMapC(f, i, W, H, lw, lh, ow, oh, pos))
                pos += Q * oh * ow
        per_frame_scores = pos // n
        d_grids = api._device_table(grids, "cuda")
        d_maps = api._device_table(maps, "cuda")
        g = HogGridsC()
        g.d_features, g.count, g.width, g.height, g.d_grids = feats.data_ptr(), len(grids), 0, 0, d_grids.data_ptr()
        scores = torch.empty(pos, dtype=torch.float32, device="cuda")

        def score():
            api._check(ctx.h, lib.sd_hog_correlate(ctx.h, C.byref(g), K, VARIANT, ptr(filt), Q, FW, FH, None, 0, 0, ptr(scores)))

        t_score = timed(score, args.reps)
        out = torch.empty((n, MAX_DET, 9), dtype=torch.int32, device="cuda")
        count = torch.empty(n, dtype=torch.int32, device="cuda")
        above = torch.empty(n, dtype=torch.int64, device="cuda")
        sample = scores[torch.randint(0, pos, (1 << 20,), device="cuda")].sort(descending=True).values
        # boxes of one frame's scores, frame-major like the scores (the comparison only): the rule's boxes as floats
        if tv is not None:
            bx = []
            for (lw, lh), (_, h, w) in levels:
                oh, ow = h - FH + 1, w - FW + 1
                y, x = torch.meshgrid(torch.arange(oh, dtype=torch.int64), torch.arange(ow, dtype=torch.int64), indexing="ij")
                x0 = (2 * x * CS * W + lw) // (2 * lw)
                x1 = (2 * (x + FW) * CS * W + lw) // (2 * lw)
                y0 = (2 * y * CS * H + lh) // (2 * lh)
                y1 = (2 * (y + FH) * CS * H + lh) // (2 * lh)
                b = torch.stack([x0, y0, x1, y1], -1).reshape(-1, 4).float()
                bx.append(b.repeat(Q, 1))
            frame_boxes = torch.cat(bx).cuda()
        for label, target in TARGETS:
            thr = float(sample[min(int(round(target / per_frame_scores * sample.numel())), sample.numel() - 1)])

            def detect():
                api._check(ctx.h, lib.sd_hog_detections(ctx.h, ptr(scores), ptr(d_maps), len(maps), n, Q, CS, FW, FH, 0, 0, thr,
                                                        OVERLAP, MAX_C, MAX_DET, ptr(out), ptr(count), ptr(above)))

            t_det = timed(detect, args.reps)
            ab = above.cpu().numpy()
            kept = count.cpu().numpy()
            t_tv = None
            if tv is not None:
                s2 = scores.view(n, per_frame_scores)

                def torch_nms():
                    masked = torch.where(s2 > thr, s2, torch.full_like(s2, -float("inf")))
                    v, idx = masked.topk(min(MAX_C, per_frame_scores), dim=1)
                    ok = v > thr
                    fr = torch.arange(n, device="cuda")[:, None].expand_as(idx)[ok]
                    keep = tv.ops.batched_nms(frame_boxes[idx[ok]], v[ok], fr, OVERLAP)
                    return fr[keep]

                t_tv = timed(torch_nms, args.reps)
            rec = {"setting": f"detect Q={Q} {label}", "frames": n, "scores_per_frame": per_frame_scores, "threshold": thr,
                   "candidates_per_frame_median": float(np.median(ab)), "candidates_per_frame_max": int(ab.max()),
                   "kept_per_frame_median": float(np.median(kept)), "detect_s": t_det, "us_per_frame": t_det / n * 1e6,
                   "pyramid_s": t_pyr, "score_s": t_score, "share_of_pyramid_and_scores": t_det / (t_pyr + t_score),
                   "comparison_only_torch_topk_batched_nms_s": t_tv, "card": info}
            print(json.dumps(rec), flush=True)
            results.append(rec)

    # end to end: frames -> detections in host arrays
    filt = torch.from_numpy(rng.normal(0, 1, (2, 3 * K + 4, FH, FW)).astype(np.float32)).cuda()
    thr = 3.0
    for Q, count_frames in [(1, n), (2, n), (2, 1)]:
        fr = frames[:count_frames]

        def e2e():
            return api.vl_hog_detect(fr, scales, filt[:Q], CS, K, thr, variant=VARIANT, overlap=OVERLAP, max_candidates=MAX_C,
                                     max_detections=MAX_DET)

        d = e2e()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            d = e2e()
        t = (time.perf_counter() - t0) / args.reps
        rec = {"setting": f"vl_hog_detect Q={Q}", "frames": count_frames, "threshold": thr, "detections": int(d.frame.size),
               "call_s": t, "frames_per_s": count_frames / t, "card": info}
        print(json.dumps(rec), flush=True)
        results.append(rec)
    if args.out:
        with open(args.out, "w") as f:
            for r in results:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
