"""Cost of ColPivHouseholderQRSolver's rank diagnostic at the feature dimensions this project trains.

    python bench_rank.py [--big] [--reps R]

Times sd_learn_rank_revealing (Gram + rank diagnostic + solve) against sd_learn (Gram + solve) on the same rows, alternating the
two, and prints one JSON line per size with the medians and their difference, the diagnostic's cost.  Sizes: D = 8,801 (the
shipped 22-landmark model) and 17,051 (config 4, N = 10,000, 44 outputs); --big adds D = 52,701 (config 5, N = 100,000, 136
outputs: about 44 GB on the device).  Rows are unit-variance features and a bias column of ones, generated on the device from a
seed, with the MatrixNorm regulariser 1.5 and the bias unregularised, as in training.  The factorisation then runs to full
rank: the worst case, since a deficient matrix stops early.  (Uncentred HOG-like rows would not: their bias column's pivot N
dwarfs the feature pivots, and at D = 52,701 the cut eps * D * N lies above them.)  The card's name and power
limit are read in the same run and printed with the figures.  Writes nothing to disk."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return name, q


def rows(N, D, M, seed):
    """[A | B] on the device, pitch a multiple of 4: A unit-variance features with a bias column, B small targets."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld = (D + M + 3) // 4 * 4
    ext = torch.empty((N, ld), dtype=torch.float32, device="cuda")
    for b in range(0, N, 4096):                       # in slices: the big config does not fit a second full-size temporary
        e = min(N, b + 4096)
        blk = torch.randn((e - b, D), generator=g, device="cuda")
        blk[:, -1] = 1.0
        ext[b:e, :D] = blk
        ext[b:e, D:D + M] = 0.05 * torch.randn((e - b, M), generator=g, device="cuda")
    return ext, ld


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--big", action="store_true", help="also D = 52,701 (config 5)")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    from superviseddescent_b200 import _capi
    from superviseddescent_b200 import api as sd
    if not torch.cuda.is_available():
        raise SystemExit("bench_rank.py needs a CUDA device")
    ctx = sd.default_context()
    lib = _capi.lib()
    name, power = card()
    sizes = [(8801, 10000, 44), (17051, 10000, 44)] + ([(52701, 100000, 136)] if args.big else [])
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    for D, N, M in sizes:
        ext, ld = rows(N, D, M, seed=D)
        X = torch.empty((D, M), dtype=torch.float32, device="cuda")
        lam = C.c_float(0)
        rank = C.c_int(-2)
        A, B = C.c_void_p(ext.data_ptr()), C.c_void_p(ext.data_ptr() + 4 * D)

        def learn():
            return lib.sd_learn(ctx.h, A, C.c_int64(ld), B, C.c_int64(ld), N, D, M, C.byref(reg), C.c_void_p(X.data_ptr()), C.byref(lam))

        def learn_rank():
            return lib.sd_learn_rank_revealing(ctx.h, A, C.c_int64(ld), B, C.c_int64(ld), N, D, M, C.byref(reg), C.c_void_p(X.data_ptr()),
                                               C.byref(lam), C.byref(rank))

        times = {"learn": [], "rank": []}
        for rep in range(args.reps + 1):                  # the first round warms up workspaces and tensor maps
            for key, fn in (("learn", learn), ("rank", learn_rank)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rc = fn()
                torch.cuda.synchronize()
                if rc:
                    raise SystemExit(f"{key} failed: {lib.sd_last_error(ctx.h).decode()}")
                if rep:
                    times[key].append(time.perf_counter() - t0)
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        print(json.dumps({"D": D, "N": N, "M": M, "rank": rank.value, "learn_s": round(med["learn"], 4),
                          "learn_rank_revealing_s": round(med["rank"], 4), "diagnostic_s": round(med["rank"] - med["learn"], 4),
                          "reps": args.reps, "gpu": name, "power_limit_and_max_sm_clock": power}), flush=True)
        del ext, X
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
