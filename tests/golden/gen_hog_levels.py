"""Generates tests/golden/hog_levels_ref.npz: fingerprints of the landmark HOG feature rows (sd_hog_batch) of the four
detect levels, which tests/test_gpu_hog_sector.py compares bit for bit.

    python tests/golden/gen_hog_levels.py        # on a GPU

Inputs: bench.py's host frames and boxes at its seed, bench.synth_frames_numpy(64, 1234) (tests/synth.smooth_images, the
frames of its CPU leg) and bench.synth_boxes(64, 1234), the shipped model's mean shape aligned to each box, and each level's
HOG parameters.  The frames of bench.py's GPU leg are not used: they come out of cuDNN convolutions, whose rounding may
depend on the algorithm the library picks.  A row is stored as the SHA-256 of its float32 bytes (the rows themselves are
9 MB) and its float64 sum, which only serves the failure message.

The committed fixture was generated on an H100 with the library built from commit 9e0f84e, the last one before the
orientation bin's sector search, so that the test compares the sector search with the rule it replaced.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "hog_levels_ref.npz")
FACES = 64
SEED = 1234


def level_rows(faces=FACES):
    """{level: (faces, D) float32 feature rows} of the levels 0..3 of the shipped model on the seeded faces."""
    import ctypes as C
    import torch
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import bench
    from superviseddescent_b200 import _capi
    from superviseddescent_b200 import api as sd
    ctx = sd.Context(0)
    model = sd.load_detection_model(bench.MODEL, ctx)
    L = model.num_landmarks
    frames = torch.from_numpy(bench.synth_frames_numpy(faces, SEED)).cuda()
    boxes = bench.synth_boxes(faces, SEED)
    x0 = torch.from_numpy(np.stack([sd.align_mean(model.get_mean(), b) for b in boxes])).cuda()
    norm = sd.NormalisationC()
    _capi.lib().sd_model_normalisation(model._m, C.byref(norm))
    ib = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), bench.W_IMG, bench.H_IMG, frames.stride(1), frames.stride(0), faces)
    rows = {}
    for level in range(4):
        hp = model.hog_param(level)
        D = _capi.lib().sd_hog_feature_length(L, C.byref(hp))
        A = torch.empty((faces, D), dtype=torch.float32, device="cuda")
        rc = _capi.lib().sd_hog_batch(ctx.h, C.byref(ib), None, _capi.ptr(x0), C.c_int64(2 * L), faces, L, C.byref(norm),
                                      C.byref(hp), _capi.ptr(A), C.c_int64(D))
        assert rc == 0, _capi.lib().sd_last_error(ctx.h)
        rows[level] = A.cpu().numpy()
    return rows


def fingerprints(rows):
    """SHA-256 of each row's float32 bytes, (faces, 32) uint8."""
    return np.stack([np.frombuffer(hashlib.sha256(np.ascontiguousarray(r, dtype=np.float32).tobytes()).digest(), dtype=np.uint8)
                     for r in rows])


if __name__ == "__main__":
    rows = level_rows()
    out = {}
    for level, r in rows.items():
        out[f"sha256_{level}"] = fingerprints(r)
        out[f"sum_{level}"] = r.astype(np.float64).sum(axis=1)
    np.savez(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items()})
