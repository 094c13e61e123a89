"""Dense HOG of whole frames (sd_hog_dense): throughput on the GPU against the reference's hog.c on every host core.

    python bench_hog_dense.py [--frames 256] [--reps 20] [--cpu-frames N] [--out FILE]

For 1280x720 and 1920x1080 grey frames (a batch of --frames per call) and three settings -- cell size 8 at K = 9 and at K = 4,
cell size 4 at K = 9, UoCTTI -- it reports the kernel time from CUDA events after warm-up, frames/s, the algorithmic traffic
(W*H bytes in, hogW*hogH*dd*4 bytes out) as GB/s and as a share of 3.35 TB/s (H100 SXM HBM3), the algorithmic flops
W*H*(24 + 4K) as TFLOP/s and as a share of 67 TFLOP/s (H100 SXM FP32, dense), which of the two bounds the kernel, and the
reference's vl_hog_put_image + vl_hog_extract (oracle/_ref) run on all host cores as the CPU figure ("not measured" when
oracle/_ref is absent).  The card's name and power limit are read in the same run.  One JSON line per setting, then a summary
line; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
FP32_FLOPS_PER_S = 67e12
SIZES = [(1280, 720), (1920, 1080)]
SETTINGS = [(8, 9, 1), (8, 4, 1), (4, 9, 1)]      # (cell size, K, variant)


def card():
    """Name, power limit and max SM clock of GPU 0, read with nvidia-smi (None when it cannot be read)."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        name, power, clock = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return None


def frames_for(n, w, h, seed):
    """n grey frames with smooth structure and noise (every gradient direction, flat areas)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = 127.5 + 90 * np.sin(x / 23.0 + np.cos(y / 31.0)) * np.cos(y / 17.0)
    out = np.empty((n, h, w), dtype=np.uint8)
    for i in range(n):
        out[i] = np.clip(np.round(np.roll(base, 7 * i, axis=1) + rng.normal(0, 10, (h, w))), 0, 255)
    return out


def cpu_reference(frames, cs, K, variant, count):
    """Frames/s of the reference's hog.c (oracle/_ref) on all host cores, or None."""
    from oracle import oracle as O
    if not O.ref_available():
        return None
    ref = O.ref()
    imgs = [np.ascontiguousarray(frames[i % len(frames)], dtype=np.float32) for i in range(min(count, len(frames)))]
    h, w = imgs[0].shape
    hw, hh = (w + cs // 2) // cs, (h + cs // 2) // cs
    dd = 3 * K + 4 if variant == 1 else 4 * K
    threads = os.cpu_count() or 1
    outs = [np.empty(dd * hh * hw, dtype=np.float32) for _ in range(threads)]

    def one(i):
        img = imgs[i % len(imgs)]
        ref.ref_vl_hog(variant, K, img.ctypes.data_as(C.POINTER(C.c_float)), w, h, cs,
                       outs[i % threads].ctypes.data_as(C.POINTER(C.c_float)), None)

    with ThreadPoolExecutor(max_workers=threads) as ex:       # ctypes releases the GIL inside the call
        list(ex.map(one, range(threads)))                      # warm-up
        t0 = time.perf_counter()
        list(ex.map(one, range(count)))
        dt = time.perf_counter() - t0
    return {"frames_per_s": count / dt, "threads": threads}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256, help="frames per call")
    ap.add_argument("--reps", type=int, default=20, help="timed calls per setting")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=0, help="frames for the CPU figure (0: four per host core)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()

    import torch
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import ImageBatchC
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_dense.py needs a CUDA device")
    ctx = api.default_context()
    lib = _capi.lib()
    info = card()
    cpu_frames = args.cpu_frames or 4 * (os.cpu_count() or 1)
    lines = []
    for (w, h) in SIZES:
        host = frames_for(args.frames, w, h, seed=w)
        dev = torch.from_numpy(host).cuda()
        ib = ImageBatchC(C.c_void_p(dev.data_ptr()), w, h, dev.stride(1), dev.stride(0), args.frames)
        for cs, K, variant in SETTINGS:
            dd, hh, hw = api.hog_dense_shape(w, h, cs, K, variant)
            out = torch.empty((args.frames, dd, hh, hw), dtype=torch.float32, device="cuda")

            def call():
                rc = lib.sd_hog_dense(ctx.h, C.byref(ib), cs, K, variant, _capi.ptr(out), None)
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
            bytes_ = args.frames * (w * h + hw * hh * dd * 4)
            flops = args.frames * w * h * (24 + 4 * K)
            t_bytes, t_flops = bytes_ / HBM_BYTES_PER_S, flops / FP32_FLOPS_PER_S
            cpu = cpu_reference(host, cs, K, variant, cpu_frames)
            rec = {
                "metric": "hog_dense", "width": w, "height": h, "cell_size": cs, "num_bins": K, "variant": variant,
                "frames_per_call": args.frames, "kernel_ms_per_call": round(ms, 4), "us_per_frame": round(1e3 * ms / args.frames, 3),
                "frames_per_s": round(args.frames / sec, 1),
                "gb_per_s": round(bytes_ / sec / 1e9, 1), "hbm_share": round(bytes_ / sec / HBM_BYTES_PER_S, 4),
                "tflop_per_s": round(flops / sec / 1e12, 2), "fp32_share": round(flops / sec / FP32_FLOPS_PER_S, 4),
                "bound": "memory" if t_bytes >= t_flops else "fp32",
                "share_of_bound": round(max(t_bytes, t_flops) / sec, 4),
                "cpu_ref_frames_per_s": round(cpu["frames_per_s"], 2) if cpu else "not measured",
                "cpu_threads": cpu["threads"] if cpu else None,
                "gpu": info if info else "not read",
            }
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            del out
        del dev
    summary = {"metric": "hog_dense_summary", "gpu": info if info else "not read",
               "frames_per_s": {f"{r['width']}x{r['height']}_cs{r['cell_size']}_K{r['num_bins']}": r["frames_per_s"] for r in lines}}
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for r in lines + [summary]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
