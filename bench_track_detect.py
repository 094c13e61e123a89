"""One face-tracking step with the detector inside it (sd_track_detect_faces) against the same step composed from the earlier
Python calls.

    python bench_track_detect.py [--frames 256] [--faces 4] [--reps 10]

Workload: --frames seeded 1280x720 grey device frames (bench_hog_filters.py's), one stream each, --faces tracks per stream
(1,024 at the defaults) from align_mean of seeded boxes, the shipped face_landmarks_model_rcr_22.bin, and a random 6 x 6-cell
filter at cell size 8, K = 9, UoCTTI.  The detector runs with detect_threshold = -inf and max_detections = 4, so that its output
size is fixed, over the pyramid 2^(-l/5) while a level holds the filter; track_overlap 0.5, keep-alive threshold 0.  Two
settings: the detector on every 8th frame (a tracker that re-scans its streams round-robin) and on every frame.  For each it
reports
  - the whole step per call, with CUDA events;
  - in a torch.profiler run of its own, the step's kernel time in phases, cut at the kernels that start each phase in launch
    order: the track step, the pyramid with scores and detections, association with compaction and merge, the new rows' cascade
    and their box scores;
  - the same step composed from the earlier calls in the same process (track_faces, vl_hog_detect of the listed frames,
    the association in numpy, detect_faces from host frames, track_boxes, hog_box_scores, the merge in numpy), on the host
    clock, with every output checked equal to the new call's.
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

from bench_hog_filters import CS, FH, FW, H, K, VARIANT, W, card, frames_for  # noqa: E402

MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")
MAX_DET, TRACK_OVERLAP = 4, 0.5
PHASES = ("track_step", "detector", "association_merge", "new_cascade", "new_box_scores")
ASSOC = ("group_count_kernel", "scan_kernel", "group_fill_kernel", "associate_kernel", "new_rows_kernel", "merge_kernel")


def phases(kernels):
    """Kernel time (ms) of one step by phase, from its (name, us) kernels in launch order: the track step ends with the first
    track_finish_kernel, the detector runs until the association's first kernel, the new rows' cascade from new_rows_kernel to
    the next track_box_kernel, and their box scores from there to the second track_finish_kernel."""
    out = dict.fromkeys(PHASES + ("copies",), 0.0)
    state, finishes = "track_step", 0
    for name, us in kernels:
        if name.startswith(("Memcpy", "Memset")):
            out["copies"] += us / 1000.0
            continue
        if any(k in name for k in ASSOC):
            out["association_merge"] += us / 1000.0
            if "new_rows_kernel" in name:
                state = "new_cascade"
            continue
        if state == "track_step" and finishes == 1:
            state = "detector"
        if state == "new_cascade" and "track_box_kernel" in name:
            state = "new_box_scores"
        out[state] += us / 1000.0
        if "track_finish_kernel" in name:
            finishes += 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--faces", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_detect.py needs a CUDA device")
    from superviseddescent_b200 import api
    import track_detect_ref

    n, per = args.frames, args.faces
    T = n * per
    m = api.load_detection_model(MODEL)
    host = frames_for(n, W, H, seed=1)
    frames = torch.from_numpy(host).cuda()
    rng = np.random.default_rng(2)
    side = rng.integers(120, 240, T)
    boxes = np.stack([rng.integers(0, W - side), rng.integers(0, H - side), side, side], 1).astype(np.int32)
    face = np.repeat(np.arange(n), per).astype(np.int32)
    prev = torch.from_numpy(np.stack([api.align_mean(m.get_mean(), b) for b in boxes])).cuda()
    filt = torch.from_numpy(np.random.default_rng(3).normal(0, 0.1, (3 * K + 4, FH, FW)).astype(np.float32)).cuda()
    ff = (filt, 0.0)
    d_face = torch.from_numpy(face).cuda()
    scales, l = [], 0
    while True:
        s = 2.0 ** (-l / 5)
        (_, _), (_, hh, hw) = api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)
        if hh < FH or hw < FW:
            break
        scales.append(s)
        l += 1
    neg = float("-inf")

    def step(listed):
        return m.track_and_detect(frames, d_face, prev, ff, (FW, FH), CS, K, 0.0, scales, listed, neg, variant=VARIANT,
                                  track_overlap=TRACK_OVERLAP, max_detections=MAX_DET)

    def composed(listed):
        old = m.track_faces(frames, d_face, prev, ff, (FW, FH), CS, K, 0.0, variant=VARIANT)
        d = api.vl_hog_detect(frames[torch.as_tensor(listed, device=frames.device)], scales, filt[None], CS, K, neg, variant=VARIANT,
                              bias=torch.zeros(1), max_detections=MAX_DET)
        ob, oa = old.boxes.cpu().numpy(), old.alive.cpu().numpy()
        det_frame = np.asarray(listed, np.int32)[d.frame]
        keep = track_detect_ref.associate(det_frame, d.boxes, face, ob, oa, TRACK_OVERLAP)
        nf, nb = det_frame[keep], d.boxes[keep]
        lm = m.detect_faces(list(host), nf, boxes=nb)
        B, valid = api.track_boxes(lm, m)
        B, valid = B.cpu().numpy(), valid.cpu().numpy()
        sc = np.full(len(nf), np.nan, np.float32)
        sc[valid] = api.hog_box_scores(frames, nf[valid], B[valid], filt, 0.0, CS, K, VARIANT).cpu().numpy()
        frame = np.concatenate([face, nf])
        bx = np.concatenate([ob, B])
        scores = np.concatenate([old.scores.cpu().numpy(), sc])
        alive = track_detect_ref.merge(frame, bx, scores, np.concatenate([oa, valid & (sc > 0)]), T, TRACK_OVERLAP)
        return np.concatenate([old.landmarks.cpu().numpy(), lm]), bx, scores, alive, frame, len(nf)

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    from torch.profiler import ProfilerActivity, profile
    results = {}
    for label, listed in (("every_8th_frame", list(range(0, n, 8))), ("every_frame", list(range(n)))):
        out = step(listed)
        want = composed(listed)
        got = [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in out]
        equal = all(np.array_equal(np.asarray(g).view(np.uint32) if np.asarray(g).dtype == np.float32 else g,
                                   np.asarray(w, np.float32).view(np.uint32) if np.asarray(g).dtype == np.float32 else w)
                    for g, w in zip(got, want))
        for _ in range(3):
            step(listed)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.reps):
            step(listed)
        e1.record()
        e1.synchronize()
        step_ms = e0.elapsed_time(e1) / args.reps
        t0 = time.perf_counter()
        for _ in range(2):
            composed(listed)
        torch.cuda.synchronize()
        composed_ms = (time.perf_counter() - t0) * 1000 / 2
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(listed)
            torch.cuda.synchronize()
        kernels = sorted(((e.time_range.start, e.name, e.time_range.elapsed_us()) for e in prof.events()
                          if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda k: k[0])
        ph = phases([(name, us) for _, name, us in kernels])
        results[label] = {
            "listed_frames": len(listed), "new_rows": out.num_new, "alive": int(out.alive.sum()),
            "step_ms": round(step_ms, 4), "phase_ms": {k: round(v, 4) for k, v in ph.items()},
            "composed_ms": round(composed_ms, 3), "outputs_equal_composed": equal,
        }
        if not equal:
            raise SystemExit(f"{label}: the step differs from the composed calls: {json.dumps(results)}")

    print(json.dumps({
        "workload": f"{n} streams 1280x720, {T} tracks, rcr_22, filter {FW}x{FH} cs {CS} K {K}, {len(scales)} scales, "
                    f"max_detections {MAX_DET}, detect_threshold -inf",
        "card": card(), **results,
    }))


if __name__ == "__main__":
    main()
