"""Per-stage cost of the star-model detector (vl_hog_part_detect's chain) on one GPU.

    python bench_hog_parts.py [--frames 64] [--reps 10] [--out FILE]

Workload: the 64-frame 1280x720 set of bench_hog_filters.py, cell size 8, K = 9, UoCTTI.  Q = 2 components (a random model
and its mirror), root filters of 6 x 6 cells, P = 8 parts of 6 x 6 part-level cells, R = 4, R = 16 and the exact transform
(R null: sd_hog_distance_transform_exact, which writes placement maps, and sd_hog_part_placements_mapped).  Root scales
0.5 * 2^(-l/5) while the root level holds the root filter; the parts are scored at twice each root scale, so the pyramid is
2^(-l/5) from 1 down.  Threshold 0 on random filters: every frame fills max_candidates = 4096 and keeps max_detections = 256,
the placements' largest load at these caps.

For every stage -- pyramid, root scores, part scores, transform, assembly, detections, placements -- the time per frame from
CUDA events around --reps calls of that stage alone, on inputs the chain produced.  The transform's algorithmic bytes are one
read and one write of every part score (8 bytes per score), plus 8 bytes of placement per score where it writes placements
(the exact route); its achieved rate is compared with the H100's 3.35 TB/s.  The card name, power limit and max SM clock are
read in the same run.  One JSON line per R."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench_hog_filters import CS, FH, FW, H, K, VARIANT, W, card, frames_for  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
Q, P, PFW, PFH = 2, 8, 6, 6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_hog_parts.py needs a CUDA device")
    from superviseddescent_b200 import _capi, api
    from superviseddescent_b200._capi import (HogDetectionC, HogGridC, HogGridsC, HogPartMapC, HogPartPlacementC, HogScoreMapC,
                                              ImageBatchC, ptr)
    lib = _capi.lib()
    ctx = api.default_context()
    n = args.frames
    info = card()
    dev = "cuda:0"
    dd = 3 * K + 4

    roots, l = [], 0
    while True:
        s = 0.5 * 2.0 ** (-l / 5)
        (_, _), (_, hh, hw) = api.hog_pyramid_shape(W, H, s, CS, K, VARIANT)
        if hh < FH or hw < FW:
            break
        roots.append(s)
        l += 1
    every = list(dict.fromkeys(roots + [2 * s for s in roots]))
    ri, pi = [every.index(s) for s in roots], [every.index(2 * s) for s in roots]
    shapes = [api.hog_pyramid_shape(W, H, s, CS, K, VARIANT) for s in every]
    per = [d * h * w for _, (d, h, w) in shapes]
    offsets = [f * sum(per) + sum(per[:i]) for f in range(n) for i in range(len(every))]
    frames = torch.from_numpy(frames_for(n, W, H, 1)).cuda()
    ib = ImageBatchC(C.c_void_p(frames.data_ptr()), W, H, W, W * H, n)
    feats = torch.empty(n * sum(per), dtype=torch.float32, device=dev)
    d_off = torch.tensor(offsets, dtype=torch.int64, device=dev)
    h_scales = (C.c_double * len(every))(*every)

    rng = np.random.default_rng(0)
    root = torch.from_numpy(rng.normal(0, 0.1, (1, dd, FH, FW)).astype(np.float32)).to(dev)
    parts = torch.from_numpy(rng.normal(0, 0.1, (P, dd, PFH, PFW)).astype(np.float32)).to(dev)
    anchors1 = np.stack([rng.integers(0, 2 * FW - PFW + 1, P), rng.integers(0, 2 * FH - PFH + 1, P)], -1)
    deform1 = np.tile(np.array([0.01, 0.0, 0.01, 0.0], np.float32), (P, 1))
    model = api.HogPartModel(root[0:1], [0.0], parts[None], anchors1[None], deform1[None], max_displacement=4)
    model = api.HogPartModel(torch.cat([model.root, model.flipped(K).root]), [0.0, 0.0],
                             torch.cat([model.parts, model.flipped(K).parts]), np.concatenate([model.anchors, model.flipped(K).anchors]),
                             np.concatenate([model.deformation, model.flipped(K).deformation]))
    rf, pf = model.root.to(dev), model.parts.reshape(Q * P, dd, PFH, PFW).to(dev)

    # tables of the chain, once
    def grid_table(levels, oh_of, out_per):
        descs, outs, pos = [], [], 0
        for f in range(n):
            for i in levels:
                _, (_, h, w) = shapes[i]
                oh, ow = oh_of(h, w)
                if oh <= 0 or ow <= 0:
                    continue
                descs.append(HogGridC(w, h, offsets[f * len(every) + i], pos))
                outs.append((f, i, oh, ow, pos))
                pos += out_per * oh * ow
        return api._device_table(descs, dev), outs, pos

    rt, rmaps, rsize = grid_table(sorted(set(ri)), lambda h, w: (h - FH + 1, w - FW + 1), Q)
    pt, pmaps, psize = grid_table(sorted(set(pi)), lambda h, w: (h - PFH + 1, w - PFW + 1), Q * P)
    rscores = torch.empty(max(rsize, 1), dtype=torch.float32, device=dev)
    pscores = torch.empty(max(psize, 1), dtype=torch.float32, device=dev)
    values = torch.empty_like(pscores)
    pplace = torch.empty((max(psize, 1), 2), dtype=torch.int32, device=dev)
    total = torch.empty_like(rscores)
    pat = {(f, i): (oh, ow, pos) for f, i, oh, ow, pos in pmaps}
    descs, sdescs = [], []
    for f, i, oh, ow, pos in rmaps:
        s = ri.index(i)
        (plw, plh), _ = shapes[pi[s]]
        ph, pw, po = pat.get((f, pi[s]), (0, 0, 0))
        (lw, lh), _ = shapes[i]
        descs.append(HogPartMapC(f, s, W, H, plw, plh, ow, oh, pw, ph, pos, po, pos))
        sdescs.append(HogScoreMapC(f, s, W, H, lw, lh, ow, oh, pos))
    ptab, stab = api._device_table(descs, dev), api._device_table(sdescs, dev)
    mc, keep_anchors = model._c(dev)
    mc_d = np.ascontiguousarray(model.deformation.reshape(-1))
    MC, MD = 4096, 256
    out = torch.empty((n, MD, len(HogDetectionC._fields_)), dtype=torch.int32, device=dev)
    count = torch.empty(n, dtype=torch.int32, device=dev)
    place = torch.empty((n, MD, P, len(HogPartPlacementC._fields_)), dtype=torch.int32, device=dev)
    gr, gp = HogGridsC(), HogGridsC()
    gr.d_features, gr.count, gr.width, gr.height, gr.d_grids = feats.data_ptr(), len(rmaps), 0, 0, rt.data_ptr()
    gp.d_features, gp.count, gp.width, gp.height, gp.d_grids = feats.data_ptr(), len(pmaps), 0, 0, pt.data_ptr()
    gv = HogGridsC()
    vt = api._device_table([HogGridC(ow, oh, pos, pos) for _, _, oh, ow, pos in pmaps], dev)
    gv.d_features, gv.count, gv.width, gv.height, gv.d_grids = pscores.data_ptr(), len(pmaps), 0, 0, vt.data_ptr()
    chk = api._check
    R_now = [4]

    def transform():
        if R_now[0] is None:
            chk(ctx.h, lib.sd_hog_distance_transform_exact(ctx.h, C.byref(gv), Q * P, C.c_void_p(mc_d.ctypes.data), ptr(values),
                                                           ptr(pplace)))
        else:
            chk(ctx.h, lib.sd_hog_distance_transform(ctx.h, C.byref(gv), Q * P, C.c_void_p(mc_d.ctypes.data), R_now[0], ptr(values),
                                                     None))

    def placements():
        if R_now[0] is None:
            chk(ctx.h, lib.sd_hog_part_placements_mapped(ctx.h, ptr(values), ptr(pplace), ptr(ptab), len(descs), C.byref(mc), CS,
                                                         ptr(out), ptr(count), n, MD, ptr(place)))
        else:
            chk(ctx.h, lib.sd_hog_part_placements(ctx.h, ptr(pscores), ptr(ptab), len(descs), C.byref(mc), C.c_void_p(mc_d.ctypes.data),
                                                  R_now[0], CS, ptr(out), ptr(count), n, MD, ptr(place)))

    stages = {
        "pyramid": lambda: chk(ctx.h, lib.sd_hog_pyramid(ctx.h, C.byref(ib), h_scales, len(every), CS, K, VARIANT, ptr(feats), ptr(d_off))),
        "root_scores": lambda: chk(ctx.h, lib.sd_hog_correlate(ctx.h, C.byref(gr), K, VARIANT, ptr(rf), Q, FW, FH, None, 0, 0, ptr(rscores))),
        "part_scores": lambda: chk(ctx.h, lib.sd_hog_correlate(ctx.h, C.byref(gp), K, VARIANT, ptr(pf), Q * P, PFW, PFH, None, 0, 0,
                                                               ptr(pscores))),
        "transform": transform,
        "assembly": lambda: chk(ctx.h, lib.sd_hog_part_scores(ctx.h, ptr(rscores), ptr(values), ptr(ptab), len(descs), C.byref(mc),
                                                              ptr(total))),
        "detections": lambda: chk(ctx.h, lib.sd_hog_detections(ctx.h, ptr(total), ptr(stab), len(sdescs), n, Q, CS, FW, FH, 0, 0, 0.0, 0.5,
                                                               MC, MD, ptr(out), ptr(count), None)),
        "placements": placements,
    }

    def timed(fn, reps):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / reps

    part_elems = psize
    lines = []
    for R in (4, 16, None):
        R_now[0] = R
        for fn in stages.values():                              # the chain once, in order: every stage's inputs exist
            fn()
        torch.cuda.synchronize()
        t = {name: timed(fn, args.reps) for name, fn in stages.items()}
        us = {k: v / n * 1e6 for k, v in t.items()}
        tr_bytes = (8.0 if R is not None else 16.0) * part_elems
        rec = {"R": R, "frames": n, "Q": Q, "P": P, "root_scales": len(roots), "pyramid_levels": len(every),
               "part_scores_per_frame": part_elems // n, "detections_per_frame": float(count.float().mean()),
               "us_per_frame": {k: round(v, 2) for k, v in us.items()},
               "transform_bytes": tr_bytes, "transform_GBps": tr_bytes / t["transform"] / 1e9,
               "transform_share_of_hbm": tr_bytes / t["transform"] / HBM_BYTES_PER_S,
               "transform_assembly_placements_us": round(us["transform"] + us["assembly"] + us["placements"], 2),
               "part_correlate_us": round(us["part_scores"], 2), "card": info}
        lines.append(rec)
        print(json.dumps(rec))
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
