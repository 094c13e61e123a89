"""Training in chunks of rows: what splitting a level costs, and a training set whose feature matrix does not fit on the GPU.

    python bench_train_chunks.py [--levels S] [--big-n 300000] [--skip-big]

Prints one JSON line per run and one header line with the card's name and power limit:
  - configs[3] (train: 10k samples, D = 17,051) and configs[4] (train5: 100k samples, D = 52,701) on one GPU, each with one chunk
    (the automatic size) and with 2 and 4 forced chunks: seconds per level, chunk count, weights checksum (sum of |X| per level);
  - configs[4]'s geometry at --big-n samples (300k: the one-shot [A | b] alone would be 63 GB): the automatic chunk count, train
    seconds, and the device memory in use after each level (torch.cuda.mem_get_info).
The training data are bench.py's synthetic sets (same generators, same seeds).  Nothing is written to the tree.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


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


def run(sd, ctx, bench, cfg, n, levels, rows_per_chunk, tag):
    import torch
    model = sd.load_detection_model(bench.MODEL, ctx)
    mean, ids, right, left = bench.train_shape_model(cfg, model)
    imgs = bench.synth_train_images(dict(cfg, n=n), 0, n, "cuda")
    x0, x_gt = bench.synth_train_landmarks(sd, mean, dict(cfg, n=n), 0, n)
    hps = [sd.HoGParam(1, cfg["cells"], cs, cfg["num_bins"], rel) for cs, rel in zip(cfg["cell_sizes"], cfg["rel"])][:levels]
    ht = sd.HogTransform(imgs, hps, ids, right, left, ctx)
    D = ht.feature_length(0)
    ld = (D + 2 * cfg["landmarks"] + 3) // 4 * 4
    norm = sd.InterEyeDistanceNormalisation(ids, right, left)

    def train(use_hps, x_gt_, x0_, rows):
        regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, cfg["lambda_factor"], False), ctx) for _ in use_hps]
        sdo = sd.SupervisedDescentOptimiser(regs, norm, ctx)
        marks, mem = [], []

        def cb(_):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks.append(e)
            free, total = torch.cuda.mem_get_info()
            mem.append(round((total - free) / 1e9, 2))
        start = torch.cuda.Event(enable_timing=True)
        start.record()
        sdo.train(x_gt_, x0_, None, ht, cb, rows_per_chunk=rows)
        torch.cuda.synchronize()
        secs = [start.elapsed_time(marks[0]) * 1e-3] + [marks[i - 1].elapsed_time(marks[i]) * 1e-3 for i in range(1, len(marks))]
        return sdo, secs, mem

    train(hps[:1], x_gt[:2048], x0[:2048], None)             # warm-up: modules, workspaces, tensor maps
    out = []
    for rows in rows_per_chunk:
        sdo, secs, mem = train(hps, x_gt, x0, rows)
        line = {"run": tag, "config": cfg["name"].split(":")[0], "samples": n, "feature_dim": D, "levels": len(hps),
                "rows_per_chunk": sdo.chunk_rows, "chunks": [math.ceil(n / r) for r in sdo.chunk_rows], "train_s": round(sum(secs), 3),
                "s_per_level": [round(s, 3) for s in secs], "weights_checksum": [float(r.x.double().abs().sum()) for r in sdo.regressors],
                "one_shot_features_gb": round(n * ld * 4 / 1e9, 1), "device_gb_in_use_after_level": mem}
        print(json.dumps(line), flush=True)
        out.append(line)
        del sdo
        torch.cuda.empty_cache()
    del ht, imgs
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, default=None, help="cascade levels per run (default: all of the config's)")
    ap.add_argument("--big-n", type=int, default=300000)
    ap.add_argument("--skip-big", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_chunks.py measures on the GPU: no CUDA device")
    import bench
    from superviseddescent_b200 import api as sd
    ctx = sd.default_context()
    print(json.dumps({"card": card()}), flush=True)
    for name in ("train", "train5"):
        cfg = bench.TRAIN_CFGS[name]
        n = cfg["n"]
        levels = args.levels or len(cfg["cell_sizes"])
        run(sd, ctx, bench, cfg, n, levels, [None, math.ceil(n / 2), math.ceil(n / 4)], "chunks")
    if not args.skip_big:
        cfg = bench.TRAIN_CFGS["train5"]
        run(sd, ctx, bench, cfg, args.big_n, args.levels or len(cfg["cell_sizes"]), [None], "beyond-memory")


if __name__ == "__main__":
    main()
