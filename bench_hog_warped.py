"""Cost of warped samples in the landmark HOG kernel (sd_hog_batch_warped) against the unwarped, TMA-staged route, and detect on
warped faces against the host workaround.

    python bench_hog_warped.py [--batch 4096] [--reps 20] [--runs 3]

Frames and boxes are bench.py's (640x480 synthetic frames generated on the GPU, one box per frame); the landmarks are the mean
shape aligned to each box.  Warped samples get a rotation uniform in +-45 degrees about their box centre at V = the frame's size,
with the same landmarks in V.  Per level of the shipped model (K = 4) and of the same levels at K = 9: CUDA-event time per launch
of both forms, alternated, `runs` times; then one torch.profiler run of each form for hog_patch_kernel alone.  Detect: faces per
second of sd_detect_faces_device_warped, of sd_detect_faces_device on the frames, and of cv2.warpAffine of every frame on the host
cores plus upload plus sd_detect_faces_device.  Training leg (config-4 sized: 909 photos x (1 original + 10 rotations) = 9,999
samples, the shipped levels at K = 9): device bytes held and seconds per sd_train_level for in-place warps against materialised
rotated copies (cv2.warpAffine), whose X must agree bit for bit.  Accuracy: the five photos of tests/golden/examples.npz rotated by
cv2 on an expanded canvas by 0 to 180 degrees, the rcr_22 IED-normalised error of detect from the rotated photo's box, without a
warp and with rotation_warp undoing the rotation (reported, not asserted).  The card's name, power limit and SM clock are read in
the same run.  Prints one JSON line; nothing is written into the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()

    import cv2
    import torch
    import bench
    from bench_hog_dense import card
    from superviseddescent_b200 import _capi
    from superviseddescent_b200 import api as sd

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ctx = sd.Context(0)
    lib = _capi.lib()
    model = sd.load_detection_model(bench.MODEL, ctx)
    B, L = args.batch, model.num_landmarks
    frames = bench.synth_frames_torch(B, 1234, dev)
    boxes = bench.synth_boxes(B, 1234)
    mean = model.get_mean()
    x0 = torch.from_numpy(np.stack([sd.align_mean(mean, b) for b in boxes])).to(dev)
    norm = sd.NormalisationC()
    lib.sd_model_normalisation(model._m, C.byref(norm))
    ib = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), bench.W_IMG, bench.H_IMG, frames.stride(1), frames.stride(0), B)
    rng = np.random.default_rng(5)
    warps = np.stack([sd.rotation_warp((b[0] + b[2] / 2, b[1] + b[3] / 2), float(rng.uniform(-45, 45))) for b in boxes])
    table = sd._warp_table(warps, None, np.array([(bench.W_IMG, bench.H_IMG)] * B), dev)

    def hog_call(hp, A, ld, warped):
        head = (ctx.h, C.byref(ib), None, _capi.ptr(x0), C.c_int64(2 * L), B, L, C.byref(norm), C.byref(hp))
        rc = lib.sd_hog_batch_warped(*head, _capi.ptr(table), _capi.ptr(A), C.c_int64(ld)) if warped else \
            lib.sd_hog_batch(*head, _capi.ptr(A), C.c_int64(ld))
        assert rc == 0, lib.sd_last_error(ctx.h)

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    levels = []
    for K in (4, 9):
        for level in range(min(4, model.num_levels)):
            hp = model.hog_param(level)
            hp.num_bins = K
            D = lib.sd_hog_feature_length(L, C.byref(hp))
            ld = (D + 3) // 4 * 4
            A = torch.empty((B, ld), dtype=torch.float32, device=dev)
            ms = {False: [], True: []}
            for warped in (False, True):
                for _ in range(3):
                    hog_call(hp, A, ld, warped)
            for _ in range(args.runs):
                for warped in (False, True):
                    torch.cuda.synchronize()
                    e0.record()
                    for _ in range(args.reps):
                        hog_call(hp, A, ld, warped)
                    e1.record()
                    torch.cuda.synchronize()
                    ms[warped].append(e0.elapsed_time(e1) / args.reps)
            kern = {}
            for warped in (False, True):
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        hog_call(hp, A, ld, warped)
                    torch.cuda.synchronize()
                tot = [e.device_time_total for e in prof.key_averages() if "hog_patch_kernel" in e.key]
                kern["warped" if warped else "unwarped"] = sum(tot) / 5 / 1000.0
            levels.append({"K": K, "level": level, "fs": hp.num_cells * hp.cell_size, "unwarped_ms": ms[False], "warped_ms": ms[True],
                           "hog_patch_kernel_ms": kern})
            del A

    # detect: warped entry, plain entry on the frames, and the host workaround (cv2.warpAffine + upload + detect)
    out = torch.empty((B, 2 * L), dtype=torch.float32, device=dev)

    def detect(warped, images=ib):
        rc = lib.sd_detect_faces_device_warped(ctx.h, model._m, C.byref(images), None, _capi.ptr(table), _capi.ptr(x0), B, _capi.ptr(out)) \
            if warped else lib.sd_detect_faces_device(ctx.h, model._m, C.byref(images), None, _capi.ptr(x0), B, _capi.ptr(out))
        assert rc == 0, lib.sd_last_error(ctx.h)
    rates = {"warped": [], "unwarped": []}
    for w in (False, True):
        detect(w)
    for _ in range(args.runs):
        for w in (False, True):
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(5):
                detect(w)
            torch.cuda.synchronize()
            rates["warped" if w else "unwarped"].append(5 * B / (time.perf_counter() - t))
    host = frames.cpu().numpy()
    cv2.setNumThreads(os.cpu_count() or 1)
    vs = np.empty_like(host)
    t = time.perf_counter()
    for i in range(B):
        cv2.warpAffine(host[i], warps[i], (bench.W_IMG, bench.H_IMG), dst=vs[i], flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    t_warp = time.perf_counter() - t
    vd = torch.from_numpy(vs).to(dev)
    ibv = sd.ImageBatchC(C.c_void_p(vd.data_ptr()), bench.W_IMG, bench.H_IMG, vd.stride(1), vd.stride(0), B)
    detect(False, ibv)
    torch.cuda.synchronize()
    ref = out.clone()
    detect(True)
    torch.cuda.synchronize()
    same = bool(torch.equal(ref.view(torch.int32), out.view(torch.int32)))
    t = time.perf_counter()
    vd.copy_(torch.from_numpy(vs))
    detect(False, ibv)
    torch.cuda.synchronize()
    t_rest = time.perf_counter() - t
    del vd, vs, host
    train = train_leg(sd, lib, ctx, model, dev, bench, cv2, torch)
    accuracy = accuracy_leg(sd, model, cv2)
    print(json.dumps({"metric": "hog_warped", "faces": B, "landmarks": L, "reps": args.reps, "levels": levels,
                      "train": train, "accuracy": accuracy,
                      "detect_faces_per_s": rates,
                      "workaround": {"cv2_warp_s": t_warp, "upload_detect_s": t_rest, "faces_per_s": B / (t_warp + t_rest),
                                     "host_threads": os.cpu_count()},
                      "warped_detect_equals_materialised": same, "card": card()}))


def train_leg(sd, lib, ctx, model, dev, bench, cv2, torch, photos=909, rotations=10):
    """sd_train_level on 909 photos x 11 samples: warps read in place against rotated copies held as frames of their own"""
    H, W, L = bench.H_IMG, bench.W_IMG, model.num_landmarks
    frames = bench.synth_frames_torch(photos, 77, dev)
    boxes = bench.synth_boxes(photos, 77)
    mean = model.get_mean()
    rng = np.random.default_rng(9)
    idx, warps, x_gt, x0 = [], [], [], []
    for f, b in enumerate(boxes):
        c = (b[0] + b[2] / 2, b[1] + b[3] / 2)
        gt = sd.align_mean(mean, b)
        for k in range(1 + rotations):
            M = np.eye(2, 3) if k == 0 else sd.rotation_warp(c, float(rng.uniform(-45, 45)))
            inv = sd.invert_warp(M)
            idx.append(f); warps.append(M)
            x_gt.append(sd.warp_landmarks(gt, inv))
            x0.append(sd.warp_landmarks(sd.align_mean(mean, b, 1 + rng.normal(0, 0.04), 1 + rng.normal(0, 0.04), rng.normal(0, 0.04),
                                                      rng.normal(0, 0.04)), inv))
    n = len(idx)
    warps = np.stack(warps)
    table = sd._warp_table(warps, None, np.array([(W, H)] * n), dev)
    host = frames.cpu().numpy()
    copies = torch.empty((n, H, W), dtype=torch.uint8, device=dev)
    for i in range(n):
        copies[i] = torch.from_numpy(cv2.warpAffine(host[idx[i]], warps[i], (W, H), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP))
    ib_own = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), W, H, frames.stride(1), frames.stride(0), photos)
    ib_cp = sd.ImageBatchC(C.c_void_p(copies.data_ptr()), W, H, copies.stride(1), copies.stride(0), n)
    d_idx = torch.tensor(idx, dtype=torch.int32, device=dev)
    xg = torch.from_numpy(np.stack(x_gt)).to(dev)
    xs = torch.from_numpy(np.stack(x0)).to(dev)
    norm = sd.InterEyeDistanceNormalisation(model.landmark_ids, ["37", "40"], ["43", "46"]).c()
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    out = {"samples": n, "photos": photos, "frame_bytes": H * W,
           "device_bytes": {"in_place": photos * H * W + n * 56, "copies": n * H * W}, "levels": []}
    for level in (0, 3):
        hp = model.hog_param(level)
        hp.num_bins = 9
        D = lib.sd_hog_feature_length(L, C.byref(hp))
        ld = (D + 2 * L + 3) // 4 * 4
        chunk = torch.empty((n, ld), dtype=torch.float32, device=dev)
        res = {}
        for which in ("in_place", "copies", "in_place", "copies"):
            f = sd.LevelFramesC(stage_half_bytes=0)
            if which == "in_place":
                f.images, f.d_sample_frame, f.d_sample_warp = C.pointer(ib_own), sd._capi.ptr(d_idx), sd._capi.ptr(table)
            else:
                f.images = C.pointer(ib_cp)
            X = torch.empty((D, 2 * L), dtype=torch.float32, device=dev)
            nxt = torch.empty_like(xs)
            torch.cuda.synchronize()
            t = time.perf_counter()
            rc = lib.sd_train_level(ctx.h, None, C.byref(f), sd._capi.ptr(xs), sd._capi.ptr(xg), n, L, C.c_int64(n), C.byref(norm), C.byref(hp),
                                    C.byref(norm), None, C.c_int64(0), C.byref(reg), 0, sd._capi.ptr(chunk), C.c_int64(ld), n, sd._capi.ptr(X),
                                    sd._capi.ptr(nxt), None)
            assert rc == 0, lib.sd_last_error(ctx.h)
            torch.cuda.synchronize()
            res.setdefault(which, []).append(time.perf_counter() - t)
            res[which + "_X"] = X.cpu().numpy()
        out["levels"].append({"level": level, "K": 9, "fs": hp.num_cells * hp.cell_size, "seconds": {k: res[k] for k in ("in_place", "copies")},
                              "X_equal": bool(np.array_equal(res["in_place_X"].view(np.uint32), res["copies_X"].view(np.uint32)))})
        del chunk
    return out


def accuracy_leg(sd, model, cv2):
    """IED-normalised error of detect on the golden photos rotated on an expanded canvas, without and with rotation_warp"""
    ex = np.load(os.path.join(ROOT, "tests", "golden", "examples.npz"))
    ids = model.landmark_ids
    sel = np.array([int(i) - 1 for i in ids])
    table = {}
    for angle in (0, 15, 30, 45, 60, 90, 180):
        plain, warped = [], []
        for i in range(5):
            g, pts, (bx, by, bw, bh) = ex[f"gray{i}"], ex[f"pts{i}"].astype(np.float64), ex["boxes"][i]
            h, w = g.shape
            R = cv2.getRotationMatrix2D((w / 2, h / 2), angle, 1.0)
            cw, ch = int(np.ceil(abs(R[0, 0]) * w + abs(R[0, 1]) * h)), int(np.ceil(abs(R[0, 1]) * w + abs(R[0, 0]) * h))
            R[0, 2] += cw / 2 - w / 2
            R[1, 2] += ch / 2 - h / 2
            rot = cv2.warpAffine(g, R, (cw, ch))
            p = pts @ R[:, :2].T + R[:, 2]
            gt = np.concatenate([p[sel, 0], p[sel, 1]]).astype(np.float32).reshape(1, -1).copy()   # a real row stride
            c = R[:, :2] @ np.array([bx + bw / 2, by + bh / 2]) + R[:, 2]
            box = np.array([[int(round(c[0] - bw / 2)), int(round(c[1] - bh / 2)), bw, bh]])
            x = model.detect_faces([rot], [0], boxes=box)
            M = sd.rotation_warp((float(c[0]), float(c[1])), -angle)
            xv = sd.warp_landmarks(model.detect_faces([rot], [0], boxes=box, warps=M[None]), M)
            for pred, acc in ((x, plain), (xv, warped)):
                e = sd.calculate_normalised_landmark_errors(pred, gt, ids, ["37", "40"], ["43", "46"])
                acc.append(float(e.mean()))
        table[str(angle)] = {"no_warp": float(np.mean(plain)), "rotation_warp": float(np.mean(warped))}
    return table


if __name__ == "__main__":
    main()
