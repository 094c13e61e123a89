"""One face-tracking step on the GPU (sd_track_faces) against the sliding-window detector it lets a video skip.

    python bench_track.py [--frames 256] [--faces 4] [--reps 20]

Workload: --frames seeded 1280x720 grey device frames (bench_hog_filters.py's), --faces faces in each (1,024 tracks at the
defaults), the shipped face_landmarks_model_rcr_22.bin, and a random 6 x 6-cell filter at cell size 8, K = 9, UoCTTI (random weights
time the same as trained ones).  Each track starts from align_mean of a seeded box.  It reports, with CUDA events, the whole step
per call and per track, and in a torch.profiler run of its own the step's kernels binned by name into rule 1 + align_mean, the
cascade (the landmark HOG and regressor kernels) and the box scores, with the step's copies and memsets in a bin of their own.
In the same process, one vl_hog_detect of the same frames (pyramid 2^(-l/5) while a level holds the filter,
scores, detections): the per-frame cost tracking avoids.  The step's landmarks are checked bit for bit against detect_faces_device
from the rule-1 boxes.  The card's name and power limit are read in the same run.  One JSON line; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_hog_filters import CS, FH, FW, H, K, VARIANT, W, card, frames_for  # noqa: E402

MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")
RULE = ("track_box_kernel",)
SCORE = ("hog_box_levels_kernel", "hog_pyramid_resize_images_kernel", "hog_dense_kernel", "correlate", "box_max_kernel",
         "track_finish_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--faces", type=int, default=4)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_track.py needs a CUDA device")
    from superviseddescent_b200 import api

    n, per = args.frames, args.faces
    T = n * per
    m = api.load_detection_model(MODEL)
    frames = torch.from_numpy(frames_for(n, W, H, seed=1)).cuda()
    rng = np.random.default_rng(2)
    side = rng.integers(120, 240, T)
    boxes = np.stack([rng.integers(0, W - side), rng.integers(0, H - side), side, side], 1).astype(np.int32)
    face = np.repeat(np.arange(n), per).astype(np.int32)
    prev = torch.from_numpy(np.stack([api.align_mean(m.get_mean(), b) for b in boxes])).cuda()
    frng = np.random.default_rng(3)
    filt = torch.from_numpy(frng.normal(0, 0.1, (3 * K + 4, FH, FW)).astype(np.float32)).cuda()
    ff = (filt, 0.0)
    d_face = torch.from_numpy(face).cuda()

    def step():
        return m.track_faces(frames, d_face, prev, ff, (FW, FH), CS, K, 0.0, variant=VARIANT)

    out = step()
    # bit identity: the step's landmarks are detect's from the rule-1 boxes
    b, valid = api.track_boxes(prev, m)
    x0 = torch.from_numpy(np.stack([api.align_mean(m.get_mean(), bb) for bb in b.cpu().numpy()])).cuda()
    ref = m.detect_batch_device(frames, x0, image_index=d_face)
    identical = bool(valid.all()) and torch.equal(out.landmarks, ref)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        step()
    e1.record()
    e1.synchronize()
    step_ms = e0.elapsed_time(e1) / args.reps

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            step()
        torch.cuda.synchronize()
    # kernels by name; the copies and memsets (detect's landmark copies, the status read-back and its reset, the bias upload) on
    # their own, so that every row is kernel time only
    phase = {"rule1_init": 0.0, "cascade": 0.0, "box_scores": 0.0, "copies": 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if us <= 0:
            continue
        name = ev.key
        key = ("copies" if name.startswith(("Memcpy", "Memset")) else "rule1_init" if any(k in name for k in RULE)
               else "box_scores" if any(k in name for k in SCORE) else "cascade")
        phase[key] += us / 1000.0 / 5
    # rule 1 runs twice per step (previous and new landmarks): the second run belongs to the box scores
    phase["box_scores"] += phase["rule1_init"] / 2
    phase["rule1_init"] /= 2

    scales, l = [], 0
    while True:
        s = 2.0 ** (-l / 5)
        (_, _), (_, hh, hw) = api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)
        if hh < FH or hw < FW:
            break
        scales.append(s)
        l += 1

    def detect():
        return api.vl_hog_detect(frames, scales, filt[None], CS, K, 0.0, variant=VARIANT)

    detect()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(3):
        detect()
    e1.record()
    e1.synchronize()
    detect_ms = e0.elapsed_time(e1) / 3

    print(json.dumps({
        "workload": f"{n} frames 1280x720, {T} tracks, rcr_22, filter {FW}x{FH} cs {CS} K {K}",
        "card": card(),
        "step_ms": round(step_ms, 4), "step_us_per_track": round(1000 * step_ms / T, 4), "tracks_per_s": round(T / step_ms * 1000),
        "phase_ms": {k: round(v, 4) for k, v in phase.items()},
        "phase_faces_per_s": {k: round(T / v * 1000) if v > 0 else None for k, v in phase.items()},
        "vl_hog_detect_ms": round(detect_ms, 4), "vl_hog_detect_ms_per_frame": round(detect_ms / n, 4),
        "alive": int(out.alive.sum()), "landmarks_bit_identical_to_detect": identical,
    }))
    if not identical:
        raise SystemExit("the step's landmarks differ from detect_faces_device from the rule-1 boxes")


if __name__ == "__main__":
    main()
