"""Colour versions of the reference's five example frames (five sizes), rebuilt from the committed grey frames and chroma.

The chroma (tests/golden/examples_chroma.npz) is the photographs' own, at a quarter of the resolution.  B and R are
grey + chroma; G is then the smallest value for which OpenCV's BGR2GRAY fixed point,
    gray = (3735 B + 19235 G + 9798 R + 2^14) >> 15,
gives the committed grey pixel back (19235 < 2^15, so one step of G never skips a grey level).  Where no G in 0..255 does,
the pixel is left grey (B = G = R).  So bgr2gray(frame) == examples["gray{i}"] exactly, and the grey frames' detect goldens
apply to the colour frames.
"""
import os

import numpy as np


def bgr_with_gray(gray, db, dr):
    """A B,G,R frame whose BGR2GRAY is `gray` exactly: B = grey + db, R = grey + dr, G as described above."""
    g = gray.astype(np.int64)
    b = np.clip(g + db, 0, 255)
    r = np.clip(g + dr, 0, 255)
    lo = g * 32768 - 3735 * b - 9798 * r - 16384           # need 19235 G >= lo
    gg = np.maximum(-(-lo // 19235), 0)
    ok = (gg <= 255) & ((3735 * b + 19235 * gg + 9798 * r + 16384) >> 15 == g)
    bgr = np.where(ok[..., None], np.stack([b, gg, r], axis=-1), g[..., None])
    return np.ascontiguousarray(bgr.astype(np.uint8))


def examples_bgr(golden):
    chroma = np.load(os.path.join(golden.dir, "examples_chroma.npz"))
    frames = []
    for i in range(5):
        gray = golden.examples[f"gray{i}"]
        h, w = gray.shape

        def up(plane):
            f = -(-h // plane.shape[0])
            return np.repeat(np.repeat(plane.astype(np.int64), f, axis=0), f, axis=1)[:h, :w]
        frames.append(bgr_with_gray(gray, up(chroma[f"db{i}"]), up(chroma[f"dr{i}"])))
    return frames
