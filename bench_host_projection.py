"""Cascade levels on a host projection: the per-row functor route against the level pipeline of HostProjection.

    python bench_host_projection.py [--levels S] [--n 20000] [--features 3000] [--cost 1] [--pose-n 100000]

Prints one header line with the card's name and power limit, then one JSON line per workload:
  - "random": a numpy projection cos(x W + b) with --features random features and a last column of ones (D = features + 1) on
    --n samples of 10 parameters; --cost repeats the feature computation to make each row dearer;
  - "pose": the pose example's projection (tests/pose_example.py, 6 parameters, D = 20) at --pose-n samples, its templates
    folded into the projection so that every route may run in chunks.
For each workload: seconds per training level on three routes -- the plain functor (rows projected one by one into a host
matrix, then learned on the GPU), HostProjection in one chunk and HostProjection in 4 chunks -- next to the seconds the host
projection alone takes over all rows (one project_host call per 48 MB batch, the staging batch of the pipeline).  The routes'
weights are reported against the functor route's (max-norm relative error).  Nothing is written to the tree.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = r.stdout.strip().splitlines()[0] if r.returncode == 0 else None
    except Exception as ex:                                  # the query is informational
        out["power_limit_and_max_sm_clock"] = repr(ex)[:100]
    return out


class RandomFeatures:
    """cos(x W_l + b_l) and a last column of ones, computed `cost` times per row (HostProjection duck type)"""

    def __init__(self, P, features, levels, cost, seed=5):
        rng = np.random.default_rng(seed)
        self.W = [rng.standard_normal((P, features)).astype(np.float32) for _ in range(levels)]
        self.b = [rng.uniform(0, 2 * np.pi, features).astype(np.float32) for _ in range(levels)]
        self.cost = cost

    def feature_length(self, level):
        return self.W[level].shape[1] + 1

    def project_host(self, x, level, first_row, out):
        for _ in range(self.cost):
            out[:, :-1] = np.cos(x @ self.W[level] + self.b[level])
        out[:, -1] = 1.0

    def row(self, x_row, level, index):
        """the same features of one row: the plain functor"""
        out = np.empty((1, self.feature_length(level)), np.float32)
        self.project_host(x_row.reshape(1, -1), level, index, out)
        return out[0]


def host_alone(proj, x, levels):
    """seconds per level of project_host over all rows, in batches of one default staging half"""
    secs = []
    for level in range(levels):
        D = proj.feature_length(level)
        ld = (D + 3) // 4 * 4
        rows = max(1, (48 << 20) // (4 * ld))
        out = np.empty((min(rows, x.shape[0]), ld), np.float32)
        t = time.perf_counter()
        for r0 in range(0, x.shape[0], rows):
            r1 = min(x.shape[0], r0 + rows)
            proj.project_host(x[r0:r1], level, r0, out[:r1 - r0, :D])
        secs.append(time.perf_counter() - t)
    return secs


def routes(sd, name, x_gt, x0, plain, piped, levels):
    import torch
    n = x_gt.shape[0]

    def train(h, rows):
        sdo = sd.SupervisedDescentOptimiser([sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False))
                                             for _ in range(levels)])
        marks = []
        torch.cuda.synchronize()
        marks.append(time.perf_counter())
        sdo.train(x_gt, x0, None, h, lambda _: (torch.cuda.synchronize(), marks.append(time.perf_counter())), rows_per_chunk=rows)
        return sdo, [round(b - a, 3) for a, b in zip(marks, marks[1:])]

    train(piped, None)                                       # warm-up: workspaces, pinned staging
    base, t_plain = train(plain, None)
    line = {"workload": name, "samples": n, "feature_dim": [piped.feature_length(l) for l in range(levels)],
            "s_per_level": {"functor": t_plain}, "weights_vs_functor": {}}
    for tag, rows in (("pipeline_1_chunk", None), ("pipeline_4_chunks", math.ceil(n / 4))):
        sdo, secs = train(piped, rows)
        line["s_per_level"][tag] = secs
        line["weights_vs_functor"][tag] = max(float(np.max(np.abs(a.x.cpu().numpy() - b.x.cpu().numpy())) / np.max(np.abs(b.x.cpu().numpy())))
                                              for a, b in zip(sdo.regressors, base.regressors))
        line.setdefault("chunk_rows", {})[tag] = sdo.chunk_rows
    line["s_per_level"]["host_projection_alone"] = [round(s, 3) for s in host_alone(piped, x0, levels)]   # on the first level's rows
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, default=2)
    ap.add_argument("--n", type=int, default=20000)
    ap.add_argument("--features", type=int, default=3000)
    ap.add_argument("--cost", type=int, default=1)
    ap.add_argument("--pose-n", type=int, default=100000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_host_projection.py measures on the GPU: no CUDA device")
    from superviseddescent_b200 import api as sd
    import pose_example as PE
    sd.default_context()
    print(json.dumps({"card": card()}), flush=True)

    rng = np.random.default_rng(9)
    x_gt = rng.uniform(-1, 1, (args.n, 10)).astype(np.float32)
    x0 = (x_gt + rng.normal(0, 0.3, x_gt.shape)).astype(np.float32)
    rf = RandomFeatures(10, args.features, args.levels, args.cost)
    routes(sd, "random", x_gt, x0, rf.row, rf, args.levels)

    x_tr, _, _ = PE.training_set(args.pose_n)
    y_tr = np.stack([PE.projection(r) for r in x_tr])
    p0 = np.zeros_like(x_tr)
    p0[:, 5] = -2000.0

    def pose(row, level, index):                              # observed = features - templates, folded into the projection
        return PE.projection(row) - y_tr[index]
    routes(sd, "pose", x_tr, p0, pose, sd.RowwiseProjection(pose, 20), args.levels)


if __name__ == "__main__":
    main()
