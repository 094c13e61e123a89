"""Dense HOG of float and multi-channel frames (sd_hog_dense_images): throughput on the GPU against the reference's hog.c on every
host core, with the 8-bit grey path (sd_hog_dense) measured in the same run.

    python bench_vl_hog.py [--frames 64] [--reps 20] [--cpu-frames N] [--lib PATH] [--out FILE]

For 1280x720 and 1920x1080 frames (a batch of --frames per call), cell size 8 and 4 at K = 9, UoCTTI, and the inputs
  u8 grey (sd_hog_dense), f32 grey, u8 3-channel interleaved (H, W, C), f32 3-channel planar (C, H, W),
each of the last three with nearest-bin and with bilinear orientations, it reports the kernel time from CUDA events after
warm-up, frames/s, the input bytes read as GB/s, and the reference's vl_hog_put_image + vl_hog_extract with the same channels and
orientation mode (oracle/_ref) run on all host cores ("not measured" when oracle/_ref is absent).  The card's name and power
limit are read in the same run.  --lib loads another build of libsd_b200.so (only its sd_hog_dense rows are run).  One JSON
line per row, then a summary line; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from bench_hog_dense import card, frames_for  # noqa: E402

SIZES = [(1280, 720), (1920, 1080)]
SETTINGS = [(8, 9, 1), (4, 9, 1)]      # (cell size, K, variant)
# (name, dtype, channels, layout); "grey_u8" runs sd_hog_dense
INPUTS = [("grey_u8", "u8", 1, "grey"), ("grey_f32", "f32", 1, "grey"), ("hwc3_u8", "u8", 3, "hwc"), ("chw3_f32", "f32", 3, "chw")]


def cpu_reference(planar, cs, K, variant, bilinear, count):
    """Frames/s of the reference's hog.c (oracle/_ref) on all host cores for (n, C, H, W) float frames, or None."""
    from oracle import vl_hog_ref
    if not vl_hog_ref.available():
        return None
    ref = vl_hog_ref.lib()
    n, c, h, w = planar.shape
    hw, hh = (w + cs // 2) // cs, (h + cs // 2) // cs
    dd = 3 * K + 4 if variant == 1 else 4 * K
    threads = os.cpu_count() or 1
    outs = [np.empty(dd * hh * hw, dtype=np.float32) for _ in range(threads)]

    def one(i):
        img = planar[i % n]
        ref.ref_vl_hog_channels(variant, K, img.ctypes.data_as(C.POINTER(C.c_float)), w, h, c, cs, int(bilinear),
                                outs[i % threads].ctypes.data_as(C.POINTER(C.c_float)), None)

    with ThreadPoolExecutor(max_workers=threads) as ex:       # ctypes releases the GIL inside the call
        list(ex.map(one, range(threads)))                      # warm-up
        t0 = time.perf_counter()
        list(ex.map(one, range(count)))
        dt = time.perf_counter() - t0
    return {"frames_per_s": count / dt, "threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64, help="frames per call")
    ap.add_argument("--reps", type=int, default=20, help="timed calls per row")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=0, help="frames for the CPU figure (0: two per host core; -1: skip)")
    ap.add_argument("--lib", default=None, help="another libsd_b200.so: time only its sd_hog_dense rows")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()

    import torch
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import HogImageC, HogImagesC, ImageBatchC
    if not torch.cuda.is_available():
        raise SystemExit("bench_vl_hog.py needs a CUDA device")
    if args.lib:
        _capi.LIB_PATH = os.path.abspath(args.lib)
    ctx = api.default_context()
    lib = _capi.lib()
    info = card()
    cpu_frames = args.cpu_frames or 2 * (os.cpu_count() or 1)
    lines = []
    for (w, h) in SIZES:
        grey = frames_for(args.frames, w, h, seed=w)
        colour = np.stack([grey, np.roll(grey, 5, axis=2), 255 - np.roll(grey, 3, axis=1)], axis=1)   # (n, 3, H, W)
        for name, dt, c, layout in INPUTS:
            if args.lib and name != "grey_u8":
                continue
            planar = colour[:, :c] if c > 1 else grey[:, None]
            host = planar.astype(np.float32) / np.float32(255) if dt == "f32" else planar
            if layout == "hwc":
                host = host.transpose(0, 2, 3, 1)
            elif layout == "grey":
                host = host[:, 0]
            dev = torch.from_numpy(np.ascontiguousarray(host)).cuda()
            if name == "grey_u8":
                ib = ImageBatchC(C.c_void_p(dev.data_ptr()), w, h, dev.stride(1), dev.stride(0), args.frames)
            else:
                s = dev.stride()
                fr = (HogImageC(w, h, 0, s[1], s[2], 0) if layout == "grey" else
                      HogImageC(w, h, 0, s[1], s[2], s[3]) if layout == "hwc" else HogImageC(w, h, 0, s[2], s[3], s[1]))
                ib = HogImagesC(C.c_void_p(dev.data_ptr()), 0 if dt == "u8" else 1, c, args.frames, fr, s[0], None)
            for cs, K, variant in SETTINGS:
                for bil in ((0,) if name == "grey_u8" else (0, 1)):
                    dd, hh, hw = api.hog_dense_shape(w, h, cs, K, variant)
                    out = torch.empty((args.frames, dd, hh, hw), dtype=torch.float32, device="cuda")

                    def call():
                        if name == "grey_u8":
                            rc = lib.sd_hog_dense(ctx.h, C.byref(ib), cs, K, variant, _capi.ptr(out), None)
                        else:
                            rc = lib.sd_hog_dense_images(ctx.h, C.byref(ib), cs, K, variant, bil, _capi.ptr(out), None)
                        if rc:
                            raise RuntimeError(lib.sd_last_error(ctx.h).decode())
                    for _ in range(args.warmup):
                        call()
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        call()
                    e1.record()
                    e1.synchronize()
                    ms = e0.elapsed_time(e1) / args.reps
                    sec = ms * 1e-3
                    bytes_in = args.frames * w * h * c * (1 if dt == "u8" else 4)
                    cpu = None
                    if args.cpu_frames >= 0 and not args.lib:
                        cpu = cpu_reference(np.ascontiguousarray(planar[:8], dtype=np.float32), cs, K, variant, bil, cpu_frames)
                    rec = {
                        "metric": "vl_hog", "input": name, "bilinear": bil, "width": w, "height": h, "cell_size": cs, "num_bins": K,
                        "variant": variant, "lib": args.lib or "tree", "frames_per_call": args.frames,
                        "kernel_ms_per_call": round(ms, 4), "us_per_frame": round(1e3 * ms / args.frames, 3),
                        "frames_per_s": round(args.frames / sec, 1), "input_gb_per_s": round(bytes_in / sec / 1e9, 1),
                        "cpu_ref_frames_per_s": round(cpu["frames_per_s"], 2) if cpu else "not measured",
                        "cpu_threads": cpu["threads"] if cpu else None,
                        "gpu": info if info else "not read",
                    }
                    print(json.dumps(rec), flush=True)
                    lines.append(rec)
                    del out
            del dev
    summary = {"metric": "vl_hog_summary", "gpu": info if info else "not read",
               "frames_per_s": {f"{r['width']}x{r['height']}_cs{r['cell_size']}_{r['input']}_bil{r['bilinear']}": r["frames_per_s"]
                                for r in lines}}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for r in lines + [summary]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
