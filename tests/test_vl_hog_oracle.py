"""The reference's own hog.c (oracle/_ref) through its multi-channel entry (oracle.vl_hog_ref): the properties of channel
selection and of the bilinear switch that the device's dense HOG of multi-channel frames relies on (tests/test_gpu_vl_hog.py)."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_ref
    vl_hog_ref.build()
    if not (oracle.ref_available() and vl_hog_ref.available()):
        pytest.skip("oracle/_ref (the reference's hog.c) is not built")
    return vl_hog_ref


def _textured(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = 127.5 + 90 * np.sin(x / 7.0 + np.cos(y / 11.0)) * np.cos(y / 5.0) + rng.normal(0, 20, (h, w))
    return np.clip(np.round(img), 0, 255).astype(np.float32)


CONFIGS = [(4, 4, 0), (8, 9, 1), (6, 9, 0), (11, 4, 1)]


@pytest.mark.parametrize("cs,K,variant", CONFIGS)
def test_one_channel_nearest_bin_is_ref_vl_hog(ref, oracle, cs, K, variant):
    import ctypes as C
    img = _textured(53, 67, cs + K)
    r = oracle.ref()
    dims = (C.c_int * 3)()
    fp = img.ctypes.data_as(C.POINTER(C.c_float))
    assert r.ref_vl_hog(variant, K, fp, 67, 53, cs, None, dims) == 0
    want = np.zeros((dims[2], dims[1], dims[0]), dtype=np.float32)
    assert r.ref_vl_hog(variant, K, fp, 67, 53, cs, want.ctypes.data_as(C.POINTER(C.c_float)), dims) == 0
    assert np.array_equal(ref.vl_hog(img, cs, K, variant), want)


@pytest.mark.parametrize("cs,K,variant", CONFIGS)
@pytest.mark.parametrize("bilinear", [False, True])
def test_identical_channels_equal_one_channel(ref, cs, K, variant, bilinear):
    img = _textured(45, 38, cs * K)
    one = ref.vl_hog(img, cs, K, variant, bilinear)
    for c in (2, 3, 16):
        assert np.array_equal(ref.vl_hog(np.stack([img] * c), cs, K, variant, bilinear), one), c


@pytest.mark.parametrize("cs,K,variant", CONFIGS)
def test_bilinear_switch_reaches_hog_c(ref, cs, K, variant):
    img = _textured(64, 80, 3)
    off = ref.vl_hog(img, cs, K, variant, False)
    on = ref.vl_hog(img, cs, K, variant, True)
    assert off.shape == on.shape and not np.array_equal(off, on)


@pytest.mark.parametrize("cs,K", [(4, 4), (8, 9), (6, 9), (11, 4)])
@pytest.mark.parametrize("bilinear", [False, True])
def test_channel_ties(ref, cs, K, bilinear):
    """Channels I and 255 - I have gradients of equal modulus and opposite sign at every pixel: the first channel keeps every
    pixel.  Opposite gradients swap the directed halves (bins k and k + K) and leave the undirected and texture dimensions."""
    img = _textured(47, 59, cs + 7 * K)
    inv = np.float32(255) - img
    hog_i = {v: ref.vl_hog(img, cs, K, v, bilinear) for v in (0, 1)}
    hog_n = {v: ref.vl_hog(inv, cs, K, v, bilinear) for v in (0, 1)}
    for v in (0, 1):
        assert np.array_equal(ref.vl_hog(np.stack([img, inv]), cs, K, v, bilinear), hog_i[v])
        assert np.array_equal(ref.vl_hog(np.stack([inv, img]), cs, K, v, bilinear), hog_n[v])
    a, b = hog_i[1], hog_n[1]                                      # UoCTTI: [directed 2K][undirected K][texture 4]
    assert np.array_equal(a[:K], b[K:2 * K]) and np.array_equal(a[K:2 * K], b[:K])
    assert np.array_equal(a[2 * K:], b[2 * K:])
    assert np.array_equal(hog_i[0], hog_n[0])                      # Dalal-Triggs: undirected only
