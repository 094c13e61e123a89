"""Kernel time of the cascade's regressor update, x <- x - (A X) (.) 1/norm(x) (sd_cascade_update: predict_rows_kernel and
gemm_finalize_kernel), at the shapes the project runs it at.

    python bench_predict.py [--reps R] [--no-big]

Shapes (N rows, D features, M = 2L outputs):
  detect   4,096 x 8,801, M = 44: one level of the detect benchmark (bench.py, 4096 faces, rcr_22 model)
  train    10,000 x 17,051, M = 44: the update of a config-4 training level
  train5   100,000 x 52,701, M = 136: the update of a config-5 training level (about 21 GB of features; --no-big skips it)

For each shape: warm-up calls, then R calls between CUDA events on the library's stream.  Printed per shape, one JSON line:
microseconds per call; achieved FMA/s (N D M useful multiply-adds) against the FP32 FMA peak at the SM clock sampled during
the timed calls (SMs x 128 lanes x clock); and the HBM floor, the time to move the operands the product needs once (A, X, x
read and x_next written) at the 3.35 TB/s of the H100 SXM data sheet.  The card's name and power limit are read in the same
run.  Inputs are generated on the device from a seed.  Writes nothing to disk."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

SHAPES = [("detect", 4096, 8801, 44), ("train", 10000, 17051, 44), ("train5", 100000, 52701, 136)]
HBM_BYTES_PER_S = 3.35e12


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return name, q


def operands(N, D, M, seed):
    """A (HOG-like: non-negative, at most 0.2, bias column of ones; pitch a multiple of 4), X, and landmarks x"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    lda = (D + 3) // 4 * 4
    A = torch.empty((N, lda), dtype=torch.float32, device="cuda")
    for b in range(0, N, 8192):                       # in slices: no second full-size temporary
        e = min(N, b + 8192)
        A[b:e] = 0.2 * torch.rand((e - b, lda), generator=g, device="cuda")
        A[b:e, D - 1] = 1.0
    X = 0.02 * torch.randn((D, M), generator=g, device="cuda")
    x = 50.0 + 100.0 * torch.rand((N, M), generator=g, device="cuda")
    return A, lda, X, x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="timed calls per shape")
    ap.add_argument("--no-big", action="store_true", help="skip the 100,000 x 52,701 shape")
    args = ap.parse_args()
    import torch
    from bench import ClockSampler
    from superviseddescent_b200 import _capi
    from superviseddescent_b200 import api as sd
    if not torch.cuda.is_available():
        raise SystemExit("bench_predict.py needs a CUDA device")
    ctx = sd.default_context()
    lib = _capi.lib()
    name, power = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for key, N, D, M in SHAPES:
        if key == "train5" and args.no_big:
            continue
        A, lda, X, x = operands(N, D, M, seed=D)
        x_next = torch.empty_like(x)
        norm = _capi.NormalisationC(1, 2, 2, (C.c_int32 * 4)(0, 1, 0, 0), (C.c_int32 * 4)(2, 3, 0, 0))

        def update():
            rc = lib.sd_cascade_update(ctx.h, _capi.ptr(A), C.c_int64(lda), N, D, _capi.ptr(X), M, _capi.ptr(x), C.byref(norm),
                                       _capi.ptr(x_next))
            if rc:
                raise SystemExit(f"sd_cascade_update failed: {lib.sd_last_error(ctx.h).decode()}")

        for _ in range(3):
            update()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        sampler = ClockSampler(0)
        sampler.start()
        e0.record(ctx.stream)                         # the context queues its work on this stream
        for _ in range(args.reps):
            update()
        e1.record(ctx.stream)
        torch.cuda.synchronize()
        clocks = sampler.stop()
        us = e0.elapsed_time(e1) * 1e3 / args.reps
        fma = float(N) * D * M
        mhz = clocks["sm_mhz"] or clocks["sm_max_mhz"]
        peak = sms * 128 * mhz * 1e6 if mhz else None
        hbm_bytes = 4.0 * (N * D + D * M + 2 * N * M)
        print(json.dumps({"shape": key, "N": N, "D": D, "M": M, "us_per_call": round(us, 1),
                          "achieved_tfma_s": round(fma / (us * 1e-6) / 1e12, 2),
                          "fp32_fma_peak_tfma_s": round(peak / 1e12, 2) if peak else None,
                          "frac_fp32_peak": round(fma / (us * 1e-6) / peak, 3) if peak else None,
                          "hbm_floor_us": round(hbm_bytes / HBM_BYTES_PER_S * 1e6, 1),
                          "reps": args.reps, "gpu": name, "power_limit_and_max_sm_clock": power, "sm_mhz_sampled": clocks["sm_mhz"],
                          "clock_event_reasons": clocks["reasons"]}), flush=True)
        del A, X, x, x_next
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
