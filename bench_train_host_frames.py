"""Training on frames that stay in host memory: the device route (frames uploaded once) against the host route (frames gathered
level by level from pinned host memory through sd_train_level), on an rcr-train-shaped set.

    python bench_train_host_frames.py [--photos 800] [--levels 5] [--big]

Workload: synthetic colour 1280x720 photos, 11 samples per photo (a face box and 10 perturbations, as apps/rcr/rcr-train.cpp
builds its set), bench.py's configs[3] HOG schedule (22 landmarks, 5 cells, 9 bins, cell sizes 11/10/8/6/6).  Prints a header line
with the card's name and power limit, then one JSON line per route: seconds per level, bytes gathered per level (host route),
device memory held for frames, and -- from a separate torch.profiler run of one host-route level -- the gather's GB/s (bytes over
the summed roi_gather_kernel time).  --big also trains on a photo set whose grey bytes exceed the card's free memory when the
host's RAM can hold it (the frames and the pinned copy the host route packs them into), and prints the measured peak host RAM.
Nothing is written to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

HOG = dict(landmarks=22, num_bins=9, cells=5, cell_sizes=[11, 10, 8, 6, 6], rel=[1.0, 0.7, 0.4, 0.25, 0.25])
W, H = 1280, 720


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = r.stdout.strip().splitlines()[0] if r.returncode == 0 else None
    except Exception:
        out["power_limit_and_max_sm_clock"] = None
    return out


def peak_rss():
    """the process's peak resident set (VmHWM of /proc/self/status) in bytes; pinned pages are resident and count"""
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmHWM:"):
                return int(line.split()[1]) * 1024
    return None


def photo_set(sd, mean, photos, seed=7):
    """photos colour frames (a few distinct textures, each photo its own buffer) and 11 samples per photo"""
    rng = np.random.default_rng(seed)
    base = [rng.integers(0, 256, (H // 8, W // 8, 3), dtype=np.uint8).repeat(8, 0).repeat(8, 1) for _ in range(4)]
    frames, x0, x_gt = [], [], []
    for i in range(photos):
        img = np.roll(base[i % 4], i % 97, axis=1).copy()
        s = int(rng.integers(220, 360))
        box = (int(rng.integers(0, W - s)), int(rng.integers(0, H - s)), s, s)
        for k in range(11):
            t = (0.0, 0.0, 1.0) if k == 0 else (rng.normal(0, 0.05), rng.normal(0, 0.05), 1 + rng.normal(0, 0.05))
            x0.append(sd.align_mean(mean, box, t[2], t[2], t[0], t[1]))
            x_gt.append(sd.align_mean(mean, box))
            frames.append(img)                               # shallow: the same array for each of the photo's samples
    return frames, np.asarray(x0, np.float32), np.asarray(x_gt, np.float32)


def run(sd, ids, frames, x0, x_gt, levels, host):
    import torch
    sd.DEVICE_FRAME_SHARE = 0.0 if host else 0.5
    hps = [sd.HoGParam(1, HOG["cells"], cs, HOG["num_bins"], rel) for cs, rel in list(zip(HOG["cell_sizes"], HOG["rel"]))[:levels]]
    ht = sd.HogTransform(frames, hps, ids, ["37", "40"], ["43", "46"])
    regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)) for _ in hps]
    sdo = sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(ids, ["37", "40"], ["43", "46"]))
    lib, ctx = sd._capi.lib(), sd.default_context()
    marks = []

    def mark(_):
        torch.cuda.synchronize()
        marks.append((time.perf_counter(), lib.sd_gathered_bytes(ctx.h)))

    torch.cuda.synchronize()
    marks.append((time.perf_counter(), lib.sd_gathered_bytes(ctx.h)))
    sdo.train(x_gt, x0, None, ht, on_training_epoch_callback=mark)
    held = 0 if ht.images is None else ht.images.numel()
    return {"route": "host" if host else "device", "samples": len(frames), "photos": len(frames) // 11,
            "seconds_per_level": [round(b[0] - a[0], 4) for a, b in zip(marks, marks[1:])],
            "bytes_gathered_per_level": [b[1] - a[1] for a, b in zip(marks, marks[1:])],
            "device_bytes_for_frames": held, "on_device": ht.on_device(),
            "weights_checksum": [float(np.abs(r.x.cpu().numpy()).sum()) for r in regs]}


def gather_rate(sd, ids, frames, x0, x_gt):
    """one host-route level under torch.profiler: bytes gathered over the summed roi_gather_kernel time"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    sd.DEVICE_FRAME_SHARE = 0.0
    ht = sd.HogTransform(frames, [sd.HoGParam(1, HOG["cells"], HOG["cell_sizes"][0], HOG["num_bins"], HOG["rel"][0])], ids, ["37", "40"], ["43", "46"])
    sdo = sd.SupervisedDescentOptimiser([sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False))],
                                        sd.InterEyeDistanceNormalisation(ids, ["37", "40"], ["43", "46"]))
    lib, ctx = sd._capi.lib(), sd.default_context()
    b0 = lib.sd_gathered_bytes(ctx.h)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        sdo.train(x_gt, x0, None, ht)
        torch.cuda.synchronize()
    nbytes = lib.sd_gathered_bytes(ctx.h) - b0
    us = sum(e.device_time_total for e in prof.key_averages() if "roi_gather_kernel" in e.key)
    return {"gather_bytes": nbytes, "gather_kernel_s": us / 1e6, "gather_GBps": round(nbytes / (us / 1e6) / 1e9, 2) if us else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--photos", type=int, default=800)
    ap.add_argument("--levels", type=int, default=5)
    ap.add_argument("--big", action="store_true")
    a = ap.parse_args()
    import torch
    from superviseddescent_b200 import api as sd
    from superviseddescent_b200 import build
    build.build()
    print(json.dumps({"card": card()}), flush=True)
    m = sd.load_detection_model(os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin"))
    ids, mean = m.landmark_ids, m.get_mean()
    frames, x0, x_gt = photo_set(sd, mean, a.photos)
    run(sd, ids, frames[:11 * 16], x0[:11 * 16], x_gt[:11 * 16], 1, True)          # warm-up of both routes' kernels
    run(sd, ids, frames[:11 * 16], x0[:11 * 16], x_gt[:11 * 16], 1, False)
    res = [run(sd, ids, frames, x0, x_gt, a.levels, host) for host in (False, True)]
    res[1]["same_weights_as_device_route"] = res[0]["weights_checksum"] == res[1]["weights_checksum"]
    res[1].update(gather_rate(sd, ids, frames, x0, x_gt))
    for r in res:
        print(json.dumps(r), flush=True)
    if a.big:
        free = torch.cuda.mem_get_info()[0]
        photos = int(free / (H * W)) + 1                         # grey bytes above the free device memory
        # the pageable colour frames, and the pinned copy the host route packs them into
        need = 2 * photos * H * W * 3
        ram = os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_AVPHYS_PAGES")
        if need > 0.8 * ram:
            print(json.dumps({"big": "not run", "photos_needed": photos, "host_bytes_needed": need, "host_bytes_available": ram}))
            return
        del frames
        frames, x0, x_gt = photo_set(sd, mean, photos)
        r = run(sd, ids, frames, x0, x_gt, 1, True)
        r["host_peak_rss_bytes"] = peak_rss()                    # measured: frames, their pinned copy and everything else
        print(json.dumps({"big": r}), flush=True)


if __name__ == "__main__":
    main()
