"""The colour example frames (tests/colour_examples.py) convert exactly to the committed grey frames and are not grey."""
import numpy as np

from colour_examples import examples_bgr


def test_colour_examples_convert_to_the_grey_frames(oracle, golden):
    frames = examples_bgr(golden)
    assert len({f.shape for f in frames}) == 5
    for i, f in enumerate(frames):
        assert f.shape[:2] == golden.examples[f"gray{i}"].shape and f.shape[2] == 3
        assert np.array_equal(oracle.bgr2gray_u8(f), golden.examples[f"gray{i}"]), i
        assert np.mean((f[..., 0] != f[..., 1]) | (f[..., 2] != f[..., 1])) > 0.9, i
