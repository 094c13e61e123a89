"""Dense HOG of caller-supplied polar gradient fields (sd_hog_dense_polar): throughput on the GPU against the reference's
vl_hog_put_polar_field on every host core, with the f32 grey rows of sd_hog_dense_images measured in the same run.

    python bench_vl_hog_polar.py [--frames 64] [--reps 20] [--warmup 3] [--cpu-frames N] [--out FILE]

For 1280x720 and 1920x1080 fields (a batch of --frames per call), cell size 8 and 4 at K = 9, UoCTTI, it times
  polar   sd_hog_dense_polar on two f32 planes, modulus and angle (the central-difference gradient of bench_hog_dense.py's frames),
          directed and undirected, nearest-bin and bilinear;
  f32     sd_hog_dense_images on the same frames as f32 grey, nearest-bin and bilinear,
and reports the kernel time from CUDA events after warm-up, frames/s, us per frame, the input bytes read as GB/s (8 B per pixel
for a polar field, 4 B for a f32 frame), and the reference's hog.c (oracle/_ref) with the same entry and orientation mode on all
host cores ("not measured" when oracle/_ref is absent).  The card's name and power limit are read in the same run.  One JSON
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
# (input, directed): polar fields both ways; f32 grey frames (sd_hog_dense_images) have no direction switch
ROWS = [("polar", 1), ("polar", 0), ("f32", None)]


def polar_of(grey):
    """(modulus, angle) float32 fields of (n, H, W) frames: the central-difference gradient, as hog.c forms it inside."""
    f = grey.astype(np.float32)
    gx = np.zeros_like(f)
    gy = np.zeros_like(f)
    gx[:, :, 1:-1] = f[:, :, 2:] - f[:, :, :-2]
    gy[:, 1:-1, :] = f[:, 2:, :] - f[:, :-2, :]
    return np.hypot(gx, gy).astype(np.float32), np.arctan2(gy, gx).astype(np.float32)


def cpu_reference(inp, fields, cs, K, variant, directed, bilinear, count):
    """Frames/s of the reference's hog.c (oracle/_ref) on all host cores, or None."""
    from oracle import vl_hog_polar_ref, vl_hog_ref
    if not (vl_hog_polar_ref.available() and vl_hog_ref.available()):
        return None
    ref = vl_hog_polar_ref.lib() if inp == "polar" else vl_hog_ref.lib()
    n, h, w = fields[0].shape
    hw, hh = (w + cs // 2) // cs, (h + cs // 2) // cs
    dd = 3 * K + 4 if variant == 1 else 4 * K
    threads = os.cpu_count() or 1
    outs = [np.empty(dd * hh * hw, dtype=np.float32) for _ in range(threads)]
    fp = C.POINTER(C.c_float)

    def one(i):
        o = outs[i % threads].ctypes.data_as(fp)
        if inp == "polar":
            m, a = fields[0][i % n], fields[1][i % n]
            ref.ref_vl_hog_polar(variant, K, m.ctypes.data_as(fp), a.ctypes.data_as(fp), w, h, directed, cs, int(bilinear), o, None)
        else:
            ref.ref_vl_hog_channels(variant, K, fields[0][i % n].ctypes.data_as(fp), w, h, 1, cs, int(bilinear), o, None)

    with ThreadPoolExecutor(max_workers=threads) as ex:       # ctypes releases the GIL inside the call
        list(ex.map(one, range(threads)))                      # warm-up
        t0 = time.perf_counter()
        list(ex.map(one, range(count)))
        dt = time.perf_counter() - t0
    return {"frames_per_s": count / dt, "threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64, help="fields per call")
    ap.add_argument("--reps", type=int, default=20, help="timed calls per row")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=0, help="fields for the CPU figure (0: two per host core; -1: skip)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()

    import torch
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import HogImageC, HogImagesC, HogPolarFieldsC
    if not torch.cuda.is_available():
        raise SystemExit("bench_vl_hog_polar.py needs a CUDA device")
    ctx = api.default_context()
    lib = _capi.lib()
    info = card()
    cpu_frames = args.cpu_frames or 2 * (os.cpu_count() or 1)
    lines = []
    for (w, h) in SIZES:
        grey = frames_for(args.frames, w, h, seed=w)
        mod, ang = polar_of(grey)
        f32 = (grey.astype(np.float32) / np.float32(255)).astype(np.float32)
        dm, da, df = (torch.from_numpy(x).cuda() for x in (mod, ang, f32))
        frame = HogImageC(w, h, 0, w, 1, 0)
        pf = HogPolarFieldsC(C.c_void_p(dm.data_ptr()), C.c_void_p(da.data_ptr()), args.frames, frame, w * h, None)
        ib = HogImagesC(C.c_void_p(df.data_ptr()), 1, 1, args.frames, frame, w * h, None)
        for cs, K, variant in SETTINGS:
            dd, hh, hw = api.hog_dense_shape(w, h, cs, K, variant)
            out = torch.empty((args.frames, dd, hh, hw), dtype=torch.float32, device="cuda")
            for inp, directed in ROWS:
                for bil in (0, 1):
                    def call():
                        if inp == "polar":
                            rc = lib.sd_hog_dense_polar(ctx.h, C.byref(pf), cs, K, variant, directed, bil, _capi.ptr(out), None)
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
                    bytes_in = args.frames * w * h * (8 if inp == "polar" else 4)
                    cpu = None
                    if args.cpu_frames >= 0:
                        src = (mod[:8], ang[:8]) if inp == "polar" else (f32[:8],)
                        cpu = cpu_reference(inp, src, cs, K, variant, directed, bil, cpu_frames)
                    rec = {
                        "metric": "vl_hog_polar", "input": inp, "directed": directed, "bilinear": bil, "width": w, "height": h,
                        "cell_size": cs, "num_bins": K, "variant": variant, "frames_per_call": args.frames,
                        "kernel_ms_per_call": round(ms, 4), "us_per_frame": round(1e3 * ms / args.frames, 3),
                        "frames_per_s": round(args.frames / sec, 1), "input_gb_per_s": round(bytes_in / sec / 1e9, 1),
                        "cpu_ref_frames_per_s": round(cpu["frames_per_s"], 2) if cpu else "not measured",
                        "cpu_threads": cpu["threads"] if cpu else None,
                        "gpu": info if info else "not read",
                    }
                    print(json.dumps(rec), flush=True)
                    lines.append(rec)
            del out
        del dm, da, df
    summary = {"metric": "vl_hog_polar_summary", "gpu": info if info else "not read",
               "frames_per_s": {f"{r['width']}x{r['height']}_cs{r['cell_size']}_{r['input']}_dir{r['directed']}_bil{r['bilinear']}":
                                r["frames_per_s"] for r in lines}}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for r in lines + [summary]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
