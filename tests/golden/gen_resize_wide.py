"""Generates tests/golden/resize_cv2_wide.npz: cv2.resize INTER_LINEAR 8UC1 pairs at the source windows and destination sizes
of the landmark HOG configuration sweep (tests/test_gpu_hog_configs.py), so that oracle.resize_linear_u8 is pinned to cv2
above the 55 px destinations of resize_cv2.npz as well.  Needs cv2 4.13 only:

    python tests/golden/gen_resize_wide.py

Each source window P x P is seeded noise (noise_source), every third one Gaussian-blurred, as in gen_golden.py; its resize to
fs x fs is stored as dst_{P}_{fs}.  Only the blurred sources are stored (blur_{P}): the noise is regenerated from its seed,
which keeps the file small.  The windows of a destination fs (sweep_windows) are P = 2 (half = 1, the
smallest window) or about 2 fs / 3, P = fs (fs + 1 when fs is odd: P is even), P = 2 fs (which cv2 computes as INTER_AREA)
and one far above fs (10 fs up to 420 px).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# destination sizes fs = num_cells * cell_size of the configuration sweep
DESTINATIONS = (4, 12, 15, 16, 30, 40, 42, 50, 55, 63, 64, 65, 72, 80, 144, 165, 180, 192)


def sweep_windows(fs):
    """The even source window sizes P that the configuration sweep resizes to fs x fs: below, equal, twice and far above fs."""
    small = 2 if fs <= 16 else (2 * fs // 3) & ~1
    return small, fs + (fs & 1), 2 * fs, min(10 * fs, 420)


def pairs():
    """{P: [fs, ...]} over every destination."""
    out = {}
    for fs in DESTINATIONS:
        for P in sweep_windows(fs):
            out.setdefault(P, []).append(fs)
    return out


def noise_source(P):
    return np.random.default_rng((20261016, P)).integers(0, 256, (P, P), dtype=np.uint8)


def main():
    import cv2
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import oracle as O
    O.build()
    g = {}
    for n, (P, dests) in enumerate(sorted(pairs().items())):
        src = noise_source(P)
        if n % 3 == 1:
            src = cv2.GaussianBlur(src, (0, 0), 1.5)
            g[f"blur_{P}"] = src
        for fs in sorted(set(dests)):
            dst = cv2.resize(src, (fs, fs))
            assert np.array_equal(dst, O.resize_linear_u8(src, fs, fs)), (P, fs)
            g[f"dst_{P}_{fs}"] = dst
    np.savez_compressed(f"{HERE}/resize_cv2_wide.npz", **g)
    print(len([k for k in g if k.startswith("dst")]), "pairs,", os.path.getsize(f"{HERE}/resize_cv2_wide.npz"), "bytes")


if __name__ == "__main__":
    main()
