"""Training a HOG filter with hard-negative mining (sd_hog_train_filter) on the GPU.

    python bench_hog_train.py [--frames 256] [--test-frames 64] [--rounds 3] [--out FILE]

Workload: --frames grey 1280x720 frames from tests/hog_train_ref.planted_frames (seed 2026): one planted object per frame at sides
48 to 160 px and four textured distractors of the same size range; cell size 8, K = 9, UoCTTI, a 6 x 6-cell filter at pad 0,
scales 2^(-l/5) while a level holds the filter; lambda 0.01, mirrored positives, 32 negatives per frame and round, mining
suppression 0.5, a cache of 16384 negatives and --rounds mining rounds.

It reports:
  - the trainer end to end (host clock around a call that ends in a synchronise) and frames/s per round;
  - per round, from the trainer's own report (sd_hog_train_report): windows mined, new, evicted, excluded, the cache size, each
    solve's Newton iterations, and the phases inside the trainer: pyramid, scores, detections and window gather by CUDA events
    around the trainer's calls, host filtering (the detections' download and the box exclusion) and the solve on the host clock,
    with the gather's bytes/s (rows read and written: 2 x rows x D x 4 bytes over its event time) -- round 0 includes the pass
    that gathers the positives;
  - the gather kernel alone on a bandwidth-sized workload: hog_windows_kernel's time from torch.profiler (no host read-back) for
    about 400 MB of rows gathered from the pyramids of 32 frames, and its bytes/s;
  - one squared-hinge solve of 20,000 of those rows (mirrored +1 against unmirrored -1), timed on the host clock;
  - the held-out VOC AP at IoU 0.5 of vl_hog_detect with the trained filter on --test-frames more frames.
The card's name and power limit are read in the same run.  One JSON line; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_hog_filters import card  # noqa: E402

W, H, CS, K, VARIANT, SIDE = 1280, 720, 8, 9, 1, 6
SLICE = 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--test-frames", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_train.py needs a CUDA device")
    import hog_train_ref as T
    from superviseddescent_b200 import api

    info = card()
    n, nt = args.frames, args.test_frames
    frames, boxes = T.planted_frames(2026, n + nt, W, H, sides=(48, 160))
    train, test = frames[:n], frames[n:]
    btrain, btest = boxes[:n], boxes[n:]
    scales = T.detector_scales(W, H, CS, SIDE)
    dev_train = torch.from_numpy(train).cuda()
    dev_test = torch.from_numpy(test).cuda()
    prm = dict(lam=0.01, flip_positives=True, negatives_per_frame=32, mine_overlap=0.5, max_negatives=16384, max_iterations=50)

    def sync_time(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, time.perf_counter() - t0

    api.train_hog_filter(dev_train[:8], np.arange(8), btrain[:8], scales, (SIDE, SIDE), CS, K, rounds=1, **prm)   # warm-up
    hf, t_total = sync_time(lambda: api.train_hog_filter(dev_train, np.arange(n), btrain, scales, (SIDE, SIDE), CS, K,
                                                         rounds=args.rounds, **prm))
    rounds = []
    for d in hf.report:
        if not d["positives"]:
            continue                                  # after an early stop
        t = d["times_ms"]
        gb = d["gathered_bytes"] / (t["gather"] * 1e-3) / 1e9 if t["gather"] > 0 else None
        rounds.append({"mined": d["mined"], "new": d["added"], "evicted": d["evicted"], "excluded": d["excluded"], "cache": d["cache"],
                       "newton_iterations": d["solve"].iterations if d["solve"] else 0, "active": d["solve"].active if d["solve"] else None,
                       "ms": {k: round(v, 3) for k, v in t.items()}, "total_ms": round(sum(t.values()), 2),
                       "frames_per_s": round(n / (sum(t.values()) * 1e-3), 1),
                       "gather_GB_per_s": round(gb, 1) if gb else None})

    # the gather kernel alone: random windows over the pyramids of 32 frames, about 400 MB of rows
    S = len(scales)
    feats, _ = api.vl_hog_pyramid(dev_train[:SLICE], scales, CS, K, VARIANT)
    maps = [m for row in feats for m in row if m is not None and m.shape[1] >= SIDE and m.shape[2] >= SIDE]
    D = 31 * SIDE * SIDE + 1
    rows_n = (400 << 20) // (D * 4)
    rng = np.random.default_rng(1)
    g = rng.integers(0, len(maps), rows_n)
    win = np.stack([g, [rng.integers(0, maps[i].shape[2] - SIDE + 1) for i in g], [rng.integers(0, maps[i].shape[1] - SIDE + 1) for i in g],
                    rng.integers(0, 2, rows_n)], 1).astype(np.int32)
    api.vl_hog_windows(maps, win, (SIDE, SIDE), K, VARIANT)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    reps = 5
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            rows = api.vl_hog_windows(maps, win, (SIDE, SIDE), K, VARIANT)
        torch.cuda.synchronize()
    kern = [e for e in prof.key_averages() if "hog_windows_kernel" in e.key]
    us = None
    if kern:
        e = kern[0]
        tot = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        us = tot / max(e.count, 1)
    gather_bytes = 2 * rows_n * D * 4
    y = torch.where(torch.from_numpy(win[:, 3]).cuda() == 1, 1.0, -1.0)[:20000]
    (w, rep), t_solve = sync_time(lambda: api.learn_squared_hinge(rows[:20000], y, 0.01, max_iterations=50))

    dt = api.vl_hog_detect(dev_test, scales, hf.filter[None], CS, K, threshold=-2.0, bias=[hf.bias], overlap=0.3, max_detections=64)
    ap_test = T.voc_ap(dt.frame, dt.boxes, dt.scores, btest)

    out = {
        "workload": {"frames": n, "test_frames": nt, "size": [W, H], "cell_size": CS, "num_bins": K, "variant": VARIANT,
                     "filter": [SIDE, SIDE], "levels": S, "rounds": args.rounds, **prm},
        "card": info,
        "trainer_s": round(t_total, 4),
        "rounds": rounds,
        "gather_kernel": {"rows": int(rows_n), "D": D, "MB": round(gather_bytes / 1e6, 1), "us": round(us, 1) if us else None,
                          "GB_per_s": round(gather_bytes / (us * 1e-6) / 1e9, 1) if us else None},
        "solve_20000_rows": {"s": round(t_solve, 4), "newton_iterations": rep.iterations, "active": rep.active},
        "held_out_ap": round(ap_test, 4),
    }
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
