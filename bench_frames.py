"""Throughput of detect on colour host frames, several faces per frame (detection_model.detect_faces).

Workloads (synthetic, seeded):
  hd4   1024 colour 1280x720 frames, four non-overlapping face boxes each (4096 faces, some over the border)
  vga1  1024 colour 640x480 frames, one face each
Arms:
  roi       detect_faces on pinned frames: the SMs gather each face's neighbourhood straight from host memory
  full      detect_faces on a pageable copy: every frame is copied to the device once and converted there
  baseline  only calls that predate detect_faces: upload the whole B,G,R frames, bgr2gray, one grey frame per face on the
            device, detect_batch_device (its align_mean runs before the timed window)
Every arm is timed with CUDA events around whole calls that end with the landmarks on the host, after a warm-up.  One JSON line
per workload: faces/s per arm, the ROI route's fallbacks, and the card's name and power limit read in the same run.

    python bench_frames.py [--steps 3] [--warmup 1] [--workloads hd4,vga1] [--arms roi,full,baseline] [--check]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")
WORKLOADS = {"hd4": (1024, 720, 1280, 4), "vga1": (1024, 480, 640, 1)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    name, limit = (r.stdout.strip().split(", ") + ["?", "?"])[:2]
    return {"name": name, "power_limit": limit}


def frames_bgr(n, h, w, seed):
    """Smooth colour frames (bilinear upsampling of coarse noise), made on the GPU, returned pinned on the host."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, h, w, 3), dtype=torch.uint8).pin_memory()
    for i in range(0, n, 64):
        k = min(64, n - i)
        coarse = torch.rand((k, 3, h // 16 + 1, w // 16 + 1), generator=g, device="cuda")
        img = F.interpolate(coarse, size=(h, w), mode="bilinear", align_corners=False)
        out[i:i + k].copy_((img * 255).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1))
    torch.cuda.synchronize()
    return out


def face_boxes(n, h, w, per_frame, seed):
    """per_frame = 1: one box per frame; 4: one box per quadrant (non-overlapping).  About a quarter hang over the border."""
    rng = np.random.default_rng(seed)
    face_frame, boxes = [], []
    cells = [(0, 0, w, h)] if per_frame == 1 else [(qx * w // 2, qy * h // 2, w // 2, h // 2) for qy in (0, 1) for qx in (0, 1)]
    for f in range(n):
        for (cx, cy, cw, ch) in cells:
            s = int(rng.integers(min(cw, ch) // 3, min(cw, ch) // 2 + 1))
            x = cx + int(rng.integers(0, cw - s + 1))
            y = cy + int(rng.integers(0, ch - s + 1))
            if rng.random() < 0.25:                       # over the frame border, on the cell's outer side
                x = x - s // 3 if cx == 0 else (x + s // 3 if cx + cw == w else x)
                y = y - s // 3 if cy == 0 else (y + s // 3 if cy + ch == h else y)
            face_frame.append(f)
            boxes.append((x, y, s, s))
    return np.array(face_frame, dtype=np.int32), np.array(boxes, dtype=np.int32)


def timed(fn, steps, warmup):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="hd4,vga1")
    ap.add_argument("--arms", default="roi,full,baseline")
    ap.add_argument("--check", action="store_true", help="assert that every arm's landmarks are bit-identical")
    args = ap.parse_args()
    from superviseddescent_b200 import api as sd
    model = sd.load_detection_model(MODEL)
    ctx = model.ctx
    arms = args.arms.split(",")
    info = card()
    for wl in args.workloads.split(","):
        n, h, w, per = WORKLOADS[wl]
        pinned = frames_bgr(n, h, w, seed=7)
        face_frame, boxes = face_boxes(n, h, w, per, seed=11)
        res = {"workload": wl, "frames": n, "size": [w, h], "faces": int(face_frame.size), "card": info}
        outs = {}
        if "roi" in arms:
            views = [pinned[i] for i in range(n)]
            fb0 = ctx.roi_fallbacks()
            outs["roi"], ms = timed(lambda: model.detect_faces(views, face_frame, boxes=boxes), args.steps, args.warmup)
            res["roi"] = {"faces_per_s": face_frame.size / (ms * 1e-3), "ms_per_call": ms,
                          "roi_fallbacks_per_call": (ctx.roi_fallbacks() - fb0) / (args.steps + args.warmup)}
        if "full" in arms:
            pageable = pinned.numpy().copy()
            frames = list(pageable)
            outs["full"], ms = timed(lambda: model.detect_faces(frames, face_frame, boxes=boxes), args.steps, args.warmup)
            res["full"] = {"faces_per_s": face_frame.size / (ms * 1e-3), "ms_per_call": ms}
            del frames, pageable
        if "baseline" in arms:
            mean = model.get_mean()
            x0 = torch.from_numpy(np.stack([sd.align_mean(mean, b) for b in boxes])).cuda()
            index = torch.from_numpy(face_frame.astype(np.int64)).cuda()

            def baseline():
                bgr = pinned.to("cuda", non_blocking=True)
                gray = sd.bgr2gray(bgr, ctx)
                return model.detect_batch_device(gray.index_select(0, index), x0).cpu().numpy()
            outs["baseline"], ms = timed(baseline, args.steps, args.warmup)
            res["baseline"] = {"faces_per_s": face_frame.size / (ms * 1e-3), "ms_per_call": ms}
            torch.cuda.empty_cache()
        if args.check:
            first = next(iter(outs.values()))
            for k, v in outs.items():
                assert np.array_equal(v, first), f"{wl}: arm {k} differs"
            res["check"] = "bit-identical: " + ",".join(outs)
        print(json.dumps(res), flush=True)
        del pinned


if __name__ == "__main__":
    main()
