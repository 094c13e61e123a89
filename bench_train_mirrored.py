"""Training on mirrored samples: each photo's samples plus their left-right mirrors, read in place from the photo
(HogTransform(mirrored=...), SD_SAMPLE_MIRRORED) against the same set built from np.fliplr copies of the photos, on the device
route and on the host route.

    python bench_train_mirrored.py [--photos 200] [--levels 5]

Workload: bench_train_host_frames.py's synthetic colour 1280x720 photos, 11 samples per photo (a face box and 10 perturbations,
as apps/rcr/rcr-train.cpp builds its set) plus their 11 mirrors (mirror_landmarks of the ground truth and of the starts), under
bench.py's configs[3] HOG schedule (22 landmarks, 5 cells, 9 bins, cell sizes 11/10/8/6/6).  Prints a header line with the card's
name and power limit, then one JSON line per (route, set): seconds per level, bytes gathered per level (host route), device memory
held for frames, and whether the weights equal the materialised set's bit for bit.  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import bench_train_host_frames as B  # noqa: E402


def mirrored_set(sd, ids, frames, x0, x_gt):
    """(frames, mirrored flags) read in place and (frames) of materialised copies, with the starts and ground truth of both"""
    perm = sd.mirror_permutation(ids)
    photos = len(frames) // 11
    x0m, xgm = sd.mirror_landmarks(x0, B.W, perm), sd.mirror_landmarks(x_gt, B.W, perm)
    flips = [np.ascontiguousarray(np.fliplr(frames[11 * p])) for p in range(photos)]
    in_place = list(frames) + list(frames)
    copies = list(frames) + [flips[i // 11] for i in range(len(frames))]
    flags = np.r_[np.zeros(len(frames), bool), np.ones(len(frames), bool)]
    return in_place, flags, copies, np.concatenate([x0, x0m]), np.concatenate([x_gt, xgm])


def run(sd, ids, frames, flags, x0, x_gt, levels, host):
    import torch
    sd.DEVICE_FRAME_SHARE = 0.0 if host else 0.5
    hps = [sd.HoGParam(1, B.HOG["cells"], cs, B.HOG["num_bins"], rel) for cs, rel in list(zip(B.HOG["cell_sizes"], B.HOG["rel"]))[:levels]]
    ht = sd.HogTransform(frames, hps, ids, ["37", "40"], ["43", "46"], mirrored=flags)
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
    return {"route": "host" if host else "device", "set": "mirrored in place" if flags is not None else "materialised copies",
            "samples": len(frames), "on_device": ht.on_device(),
            "seconds_per_level": [round(b[0] - a[0], 4) for a, b in zip(marks, marks[1:])],
            "bytes_gathered_per_level": [b[1] - a[1] for a, b in zip(marks, marks[1:])],
            "device_bytes_for_frames": held}, [r.x.cpu().numpy() for r in regs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--photos", type=int, default=200)
    ap.add_argument("--levels", type=int, default=5)
    a = ap.parse_args()
    from superviseddescent_b200 import api as sd
    from superviseddescent_b200 import build
    build.build()
    print(json.dumps({"card": B.card()}), flush=True)
    m = sd.load_detection_model(os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin"))
    ids, mean = m.landmark_ids, m.get_mean()
    frames, x0, x_gt = B.photo_set(sd, mean, a.photos)
    in_place, flags, copies, x0s, xgs = mirrored_set(sd, ids, frames, x0, x_gt)
    warm = slice(0, 11 * 8)
    w_place, w_flags, w_copies, w_x0, w_xg = mirrored_set(sd, ids, frames[warm], x0[warm], x_gt[warm])
    for host in (False, True):                                   # warm-up of every route's kernels
        run(sd, ids, w_place, w_flags, w_x0, w_xg, 1, host)
        run(sd, ids, w_copies, None, w_x0, w_xg, 1, host)
    for host in (False, True):
        r_in, w_in = run(sd, ids, in_place, flags, x0s, xgs, a.levels, host)
        r_cp, w_cp = run(sd, ids, copies, None, x0s, xgs, a.levels, host)
        r_in["same_weights_as_copies"] = all(np.array_equal(p.view(np.uint32), q.view(np.uint32)) for p, q in zip(w_in, w_cp))
        print(json.dumps(r_in), flush=True)
        print(json.dumps(r_cp), flush=True)


if __name__ == "__main__":
    main()
