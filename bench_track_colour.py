"""One face-tracking step on colour video (sd_track_detect_faces_images through detection_model.track_and_detect(multichannel=True))
against the grey step on the same frames' grey, and against the colour step composed from the earlier Python calls.

    python bench_track_colour.py [--frames 256] [--faces 4] [--reps 10]

Workload: --frames seeded 1280x720 B,G,R device frames (three of bench_hog_filters.py's grey frames as channels), one stream
each, --faces tracks per stream (1,024 at the defaults) from align_mean of seeded boxes, the shipped face_landmarks_model_rcr_22.bin,
and a random 6 x 6-cell colour filter at cell size 8, K = 9, UoCTTI.  The detector settings are bench_track_detect.py's
(detect_threshold -inf, max_detections 4, the pyramid 2^(-l/5), track_overlap 0.5, keep-alive threshold 0), on every 8th frame
and on every frame.  For each it reports
  - the colour step per call (the grey frames for the cascade made on the device by sd_bgr2gray_images inside the call) and
    the grey step on the frames' grey (bgr2gray once, outside the timing), alternated in one process, with CUDA events;
  - in a torch.profiler run of its own, the colour step's kernel time in bench_track_detect.py's phases, plus the conversion;
  - the colour step composed from the earlier calls (track_faces with multichannel, vl_hog_detect(multichannel=True) of the
    listed frames, the association in numpy, detect_faces from the grey frames, track_boxes, hog_box_scores(multichannel=True),
    the merge in numpy), on the host clock, with every output checked equal to the step's;
  - the bytes a step puts on the device for host frames, from the shapes: one colour upload, against a grey and a colour one.
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
from bench_track_detect import MAX_DET, MODEL, TRACK_OVERLAP, phases  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--faces", type=int, default=4)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_colour.py needs a CUDA device")
    from superviseddescent_b200 import api
    import track_detect_ref

    n, per = args.frames, args.faces
    T = n * per
    m = api.load_detection_model(MODEL)
    colour = torch.stack([torch.from_numpy(frames_for(n, W, H, seed=s)).cuda() for s in (1, 11, 21)], dim=3).contiguous()
    grey = api.bgr2gray(colour)
    grey_host = list(grey.cpu().numpy())
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

    def step(frames, listed, **kw):
        return m.track_and_detect(frames, d_face, prev, ff, (FW, FH), CS, K, 0.0, scales, listed, neg, variant=VARIANT,
                                  track_overlap=TRACK_OVERLAP, max_detections=MAX_DET, **kw)

    def composed(listed):
        old = m.track_faces(colour, d_face, prev, ff, (FW, FH), CS, K, 0.0, variant=VARIANT, multichannel=True)
        d = api.vl_hog_detect(colour[torch.as_tensor(listed, device=colour.device)], scales, filt[None], CS, K, neg, variant=VARIANT,
                              bias=torch.zeros(1), max_detections=MAX_DET, multichannel=True)
        ob, oa = old.boxes.cpu().numpy(), old.alive.cpu().numpy()
        det_frame = np.asarray(listed, np.int32)[d.frame]
        keep = track_detect_ref.associate(det_frame, d.boxes, face, ob, oa, TRACK_OVERLAP)
        nf, nb = det_frame[keep], d.boxes[keep]
        lm = m.detect_faces(grey_host, nf, boxes=nb)
        B, valid = api.track_boxes(lm, m)
        B, valid = B.cpu().numpy(), valid.cpu().numpy()
        sc = np.full(len(nf), np.nan, np.float32)
        sc[valid] = api.hog_box_scores(colour, nf[valid], B[valid], filt, 0.0, CS, K, VARIANT, multichannel=True).cpu().numpy()
        frame = np.concatenate([face, nf])
        bx = np.concatenate([ob, B])
        scores = np.concatenate([old.scores.cpu().numpy(), sc])
        alive = track_detect_ref.merge(frame, bx, scores, np.concatenate([oa, valid & (sc > 0)]), T, TRACK_OVERLAP)
        return np.concatenate([old.landmarks.cpu().numpy(), lm]), bx, scores, alive, frame, len(nf)

    def same(g, w):
        if isinstance(g, int):
            return g == w
        g = np.asarray(g)
        w = np.asarray(w, g.dtype)
        return g.shape == w.shape and np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                                     w.view(np.uint32) if w.dtype == np.float32 else w)

    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    from torch.profiler import ProfilerActivity, profile
    results = {}
    for label, listed in (("every_8th_frame", list(range(0, n, 8))), ("every_frame", list(range(n)))):
        out = step(colour, listed, multichannel=True)
        want = composed(listed)
        got = [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in out]
        equal = all(same(g, w) for g, w in zip(got, want))
        for _ in range(3):
            step(colour, listed, multichannel=True)
            step(grey, listed)
        colour_ms, grey_ms = [], []
        for _ in range(args.reps):                 # alternated: one colour step, one grey step
            torch.cuda.synchronize()
            e[0].record()
            step(colour, listed, multichannel=True)
            e[1].record()
            step(grey, listed)
            e[2].record()
            e[2].synchronize()
            colour_ms.append(e[0].elapsed_time(e[1]))
            grey_ms.append(e[1].elapsed_time(e[2]))
        t0 = time.perf_counter()
        composed(listed)
        torch.cuda.synchronize()
        composed_ms = (time.perf_counter() - t0) * 1000
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step(colour, listed, multichannel=True)
            torch.cuda.synchronize()
        kernels = sorted(((ev.time_range.start, ev.name, ev.time_range.elapsed_us()) for ev in prof.events()
                          if ev.device_type == torch.autograd.DeviceType.CUDA), key=lambda k: k[0])
        conv = sum(us for _, name, us in kernels if "bgr2gray_images_kernel" in name) / 1000.0
        ph = phases([(name, us) for _, name, us in kernels if "bgr2gray_images_kernel" not in name])
        results[label] = {
            "listed_frames": len(listed), "new_rows": out.num_new, "alive": int(out.alive.sum()),
            "colour_step_ms": {"median": round(float(np.median(colour_ms)), 4), "min": round(min(colour_ms), 4),
                               "max": round(max(colour_ms), 4)},
            "grey_step_ms": {"median": round(float(np.median(grey_ms)), 4), "min": round(min(grey_ms), 4), "max": round(max(grey_ms), 4)},
            "colour_phase_ms": {"bgr2gray": round(conv, 4), **{k: round(v, 4) for k, v in ph.items()}},
            "composed_colour_ms": round(composed_ms, 3), "outputs_equal_composed": bool(equal),
        }
        if not equal:
            raise SystemExit(f"{label}: the colour step differs from the composed calls: {json.dumps(results)}")

    print(json.dumps({
        "workload": f"{n} streams 1280x720 BGR, {T} tracks, rcr_22, colour filter {FW}x{FH} cs {CS} K {K}, {len(scales)} scales, "
                    f"max_detections {MAX_DET}, detect_threshold -inf",
        "upload_bytes_per_step": {"one_colour_upload": n * H * W * 3, "grey_and_colour_uploads": n * H * W * 4},
        "card": card(), **results,
    }))


if __name__ == "__main__":
    main()
