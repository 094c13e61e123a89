"""Aligned face chips (sd_face_chips through face_chips) on device frames, against cv2.warpAffine on all host cores.

    python bench_face_chips.py [--frames 256] [--faces 1024] [--reps 20]

Workload: --frames seeded 1280x720 B,G,R device frames (three of bench_hog_filters.py's grey frames as channels), --faces faces
spread evenly over them, each the align_mean of a seeded box (sides 120 to 240 px) of the shipped face_landmarks_model_rcr_22.bin's
mean, rotated about the box centre by up to +-30 degrees.  Chips are 112x112 and 224x224 on the default template (padding 0.25,
every landmark), from 8-bit frames and from the same frames as float32 in [0, 1].  For each it reports
  - ms per call and chips/s over --reps calls after warm-up, with CUDA events;
  - in a torch.profiler run of its own, the fit and warp kernel times;
  - the algorithmic bytes -- chip bytes written plus the distinct source pixels (all channels) each chip's taps touch, computed
    here from the transforms -- over the kernel time, against the H100's 3.35 TB/s of HBM3: the warp is a gather whose bytes are
    the bound that applies, as it has no arithmetic to speak of;
  - cv2.warpAffine(INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT, 0) of the same chips on every host core (one cv2 thread per
    worker), timed on the host clock, with every chip compared bit for bit to the device's.
The card's name and power limit are read in the same run.  One JSON line per configuration; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_hog_filters import H, W, card, frames_for  # noqa: E402

MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")
HBM_BYTES_PER_S = 3.35e12


def faces(mean, n, per_frame_count, seed):
    """(face_frame, landmarks (n, 2L) float32): align_mean of seeded boxes, rotated about the box centre by up to 30 degrees."""
    rng = np.random.default_rng(seed)
    mean = np.asarray(mean, np.float32).ravel()
    L = mean.size // 2
    side = rng.integers(120, 240, n)
    bx, by = rng.integers(0, W - side), rng.integers(0, H - side)
    t = rng.uniform(-np.pi / 6, np.pi / 6, n)
    x = ((mean[None, :L] + np.float32(0.5)) * side[:, None] + bx[:, None]).astype(np.float64)
    y = ((mean[None, L:] + np.float32(0.5)) * side[:, None] + by[:, None]).astype(np.float64)
    cx, cy = (bx + side / 2)[:, None], (by + side / 2)[:, None]
    c, s = np.cos(t)[:, None], np.sin(t)[:, None]
    rx, ry = cx + c * (x - cx) - s * (y - cy), cy + s * (x - cx) + c * (y - cy)
    return (np.arange(n) % per_frame_count).astype(np.int32), np.concatenate([rx, ry], 1).astype(np.float32)


def touched_pixels(c2f, size):
    """Distinct source pixels inside the frame that each chip's four taps read, summed over chips (face_chip_ref's taps)."""
    import face_chip_ref
    total = 0
    for M in c2f:
        t = face_chip_ref.taps(M, size, size, W, H)
        (ys, xs), _ = t
        mask = np.zeros((H + 1, W + 1), bool)
        for dy in (0, 1):
            for dx in (0, 1):
                yy, xx = ys + dy, xs + dx
                ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
                mask[yy[ok], xx[ok]] = True
        total += int(mask.sum())
    return total


def cpu_chips(frames_host, ff, c2f, size):
    """cv2.warpAffine of every chip on all host cores -> (seconds, chips)."""
    import cv2
    cv2.setNumThreads(1)

    def one(i):
        return cv2.warpAffine(frames_host[ff[i]], c2f[i], (size, size), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                              borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        list(ex.map(one, range(min(64, len(ff)))))      # warm-up
        t0 = time.perf_counter()
        out = list(ex.map(one, range(len(ff))))
        return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--faces", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_face_chips.py needs a CUDA device")
    from superviseddescent_b200 import api

    m = api.load_detection_model(MODEL)
    u8 = torch.stack([torch.from_numpy(frames_for(args.frames, W, H, seed=s)).cuda() for s in (1, 11, 21)], dim=3).contiguous()
    f32 = (u8.float() / 255).contiguous()
    ff, x = faces(m.get_mean(), args.faces, args.frames, seed=2)
    dff, dx = torch.from_numpy(ff).cuda(), torch.from_numpy(x).cuda()
    info = card()
    for size in (112, 224):
        tm = api.face_chip_template(m, size)
        touched = None
        for name, frames in (("u8", u8), ("f32", f32)):
            run = lambda: api.face_chips(frames, dff, dx, size, tm, channels_last=True)
            for _ in range(3):
                r = run()
            torch.cuda.synchronize()
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.reps):
                run()
            stop.record()
            stop.synchronize()
            ms = start.elapsed_time(stop) / args.reps

            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    run()
                torch.cuda.synchronize()
            kern = {"fit": 0.0, "warp": 0.0}
            for e in prof.key_averages():
                for k in kern:
                    if f"face_chip_{k}_kernel" in e.key:
                        kern[k] += e.device_time_total / 1e3 / args.reps    # us -> ms per call
            c2f = r.chip_to_frame.cpu().numpy()
            assert bool(r.valid.all())
            if touched is None:
                touched = touched_pixels(c2f, size)
            es = r.chips.element_size()
            chip_bytes = r.chips.numel() * es
            alg_bytes = chip_bytes + touched * 3 * es
            kernel_ms = kern["fit"] + kern["warp"]

            host = [f for f in frames.cpu().numpy()]
            cpu_s, cpu_out = cpu_chips(host, ff, c2f, size)
            dev = r.chips.cpu().numpy()
            equal = all(np.array_equal(dev[i].view(np.uint8), np.ascontiguousarray(cpu_out[i]).reshape(dev[i].shape).view(np.uint8))
                        for i in range(len(ff)))
            print(json.dumps({
                "bench": "face_chips", "card": info, "frames": args.frames, "faces": args.faces, "chip": size, "dtype": name,
                "ms_per_call": round(ms, 4), "chips_per_s": round(args.faces / ms * 1e3),
                "kernel_ms": {k: round(v, 4) for k, v in kern.items()},
                "alg_bytes": alg_bytes, "chip_bytes": chip_bytes, "source_bytes": touched * 3 * es,
                "alg_tb_per_s": round(alg_bytes / (kernel_ms * 1e-3) / 1e12, 3) if kernel_ms else None,
                "share_of_hbm": round(alg_bytes / (kernel_ms * 1e-3) / HBM_BYTES_PER_S, 3) if kernel_ms else None,
                "bound": "bytes (HBM)",
                "cpu_ms": round(cpu_s * 1e3, 2), "cpu_threads": os.cpu_count(), "cpu_equal_bit_for_bit": equal}), flush=True)


if __name__ == "__main__":
    main()
