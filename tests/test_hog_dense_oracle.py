"""The oracle's restatement of VLFeat's HOG (oracle.hog_core) against the reference's own hog.c (oracle/_ref) on whole frames of
sizes that are not square and not multiples of the cell size: the CPU side of the dense HOG's parity (tests/test_gpu_hog_dense.py
compares the device against both).  Bit for bit: the restatement is the reference's arithmetic in the reference's order."""
import numpy as np
import pytest


@pytest.mark.parametrize("h,w", [(29, 37), (4, 4), (479, 641), (7, 5)])
@pytest.mark.parametrize("K", [4, 9])
@pytest.mark.parametrize("variant", [0, 1])
def test_hog_core_equals_reference_hog_on_whole_frames(oracle, h, w, K, variant):
    if not oracle.ref_available():
        pytest.skip("oracle/_ref (the reference's hog.c) is not built")
    rng = np.random.default_rng(h * 1000 + w + K)
    frame = rng.integers(0, 256, size=(h, w)).astype(np.float32)
    frame[: h // 2] = np.round(frame[: h // 2] * 0.1)             # low-contrast half: small gradients, ties, zero gradients
    for cs in (4, 6, 8, 11):
        if (w + cs // 2) // cs == 0 or (h + cs // 2) // cs == 0:
            continue
        a = oracle.hog_core(frame, cs, K, variant)
        b = oracle.hog_core(frame, cs, K, variant, use_ref=True)
        assert a.shape == b.shape == (oracle.hog_dimension(variant, K), (h + cs // 2) // cs, (w + cs // 2) // cs)
        assert np.array_equal(a, b), (h, w, cs, K, variant)
