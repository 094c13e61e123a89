"""Generates tests/golden/examples_chroma.npz: the colour of the reference's five annotated example photographs, compactly.

    python tests/golden/gen_examples_chroma.py REFERENCE_DIR

The grey frames are already committed (examples.npz, gray0..gray4 = cv2 BGR2GRAY of the photographs).  What colour adds is
stored here as two signed chroma planes per photograph, B - grey and R - grey, averaged over 4 x 4 pixel blocks (cv2 INTER_AREA)
and rounded to int8: db0..db4, dr0..dr4.  tests/colour_examples.py rebuilds full-size colour frames from them whose BGR2GRAY
conversion is exactly the committed grey frame, so the detect goldens of the grey frames hold for them.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FACTOR = 4


def main(ref):
    import cv2
    ex = np.load(f"{HERE}/examples.npz")
    out = {}
    for i in range(5):
        bgr = cv2.imread(f"{ref}/examples/data/ibug_lfpw_trainset/image_000{i + 1}.png")
        gray = ex[f"gray{i}"]
        assert np.array_equal(cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY), gray)
        h, w = gray.shape
        size = ((w + FACTOR - 1) // FACTOR, (h + FACTOR - 1) // FACTOR)
        for c, name in ((0, "db"), (2, "dr")):
            diff = bgr[:, :, c].astype(np.float32) - gray.astype(np.float32)
            out[f"{name}{i}"] = np.clip(np.round(cv2.resize(diff, size, interpolation=cv2.INTER_AREA)), -127, 127).astype(np.int8)
    np.savez_compressed(f"{HERE}/examples_chroma.npz", **out)
    print("examples_chroma.npz", os.path.getsize(f"{HERE}/examples_chroma.npz"), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
