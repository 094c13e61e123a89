"""sd_hog_render (vl_hog_render) and sd_hog_relayout (flip by vl_hog_get_permutation, transpose) on the device.

  - Render: bit for bit the image of the reference's own vl_hog_render for the same features and the same non-zero starting
    image with one NaN pixel (NaN compared by position: the device writes the canonical NaN, x86 keeps the input's payload),
    for K 1 / 4 / 9 / 16, both variants, transposed glyphs or not, grids from 1 x 1 to 240 x 135 cells, HOG features and
    random signed filters; a batch of grids of mixed sizes renders each grid as it renders alone.
  - Relayout: flip and transpose are numpy's gathers with hog.c's permutation, bit for bit; flip twice is the identity.
  - Property: the HOG of a mirrored frame is the flip of the frame's HOG, to a tolerance (see test_flip_is_the_hog_of_the_mirror)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_api_ref
    vl_hog_api_ref.build()
    if not vl_hog_api_ref.available():
        pytest.skip("oracle/_ref (the reference's hog.c) is not built")
    return vl_hog_api_ref


def _grids(t, count, w, h, table=None):
    from superviseddescent_b200._capi import HogGridsC
    g = HogGridsC()
    g.d_features, g.count, g.width, g.height = t.data_ptr(), count, w, h
    g.d_grids = table.data_ptr() if table is not None else None
    return g


def _render_into(sd, feats, start, K, variant, transposed):
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    f = torch.from_numpy(np.ascontiguousarray(feats)).cuda()
    img = torch.from_numpy(start.copy()).cuda()
    dd, h, w = feats.shape
    rc = _capi.lib().sd_hog_render(ctx.h, C.byref(_grids(f, 1, w, h)), K, variant, int(transposed), _capi.ptr(img))
    assert rc == 0, _capi.lib().sd_last_error(ctx.h)
    return img.cpu().numpy()


def _relayout(sd, feats, K, variant, flip, transpose):
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    f = torch.from_numpy(np.ascontiguousarray(feats)).cuda()
    b, dd, h, w = feats.shape
    out = torch.empty_like(f)
    rc = _capi.lib().sd_hog_relayout(ctx.h, C.byref(_grids(f, b, w, h)), K, variant, flip, transpose, _capi.ptr(out))
    assert rc == 0, _capi.lib().sd_last_error(ctx.h)
    out = out.cpu().numpy()
    return out.reshape(b, dd, w, h) if transpose else out


def _hog_features(sd, w, h, K, variant, seed):
    """HOG features of a w x h cell grid: the dense HOG of a random float frame of w * 8 x h * 8 pixels."""
    rng = np.random.default_rng(seed)
    frame = rng.uniform(0, 255, (h * 8, w * 8)).astype(np.float32)
    return sd.vl_hog(frame[None], 8, K, variant)[0].cpu().numpy()


def _same(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.nan_to_num(a).view(np.uint32), np.nan_to_num(b).view(np.uint32))


CASES = [(K, v, t) for K in (1, 4, 9, 16) for v in (0, 1) for t in (0, 1)]
SIZES = [(1, 1), (3, 2), (17, 11), (240, 135)]


@pytest.mark.parametrize("K,variant,transposed", CASES)
def test_render_is_hog_c(sd, ref, K, variant, transposed):
    i = CASES.index((K, variant, transposed))
    rng = np.random.default_rng(100 + i)
    dd = 3 * K + 4 if variant else 4 * K
    for j, (w, h) in enumerate([SIZES[i % 4], SIZES[(i + 1) % 4]]):
        signed = (rng.standard_normal((dd, h, w)) * 0.5).astype(np.float32)
        feats = [signed] + ([_hog_features(sd, w, h, K, variant, i)] if j == 0 else [])
        for f in feats:
            start = rng.uniform(-0.3, 0.3, (h * 21, w * 21)).astype(np.float32)
            start.flat[start.size // 3] = np.nan
            got = _render_into(sd, f, start, K, variant, transposed)
            want = ref.Hog(variant, K, bool(transposed)).render(f, start)
            assert np.isnan(got.flat[start.size // 3])
            assert _same(got, want), (w, h, float(np.nanmax(np.abs(got - want))))


def test_render_python_and_batch_independence(sd, ref):
    """vl_hog_render of a list of grids of mixed sizes (one descriptor table) and of a batch give each grid's lone render, which
    is hog.c's render into a zeroed image."""
    rng = np.random.default_rng(7)
    K, variant = 9, 1
    grids = [rng.standard_normal((31, h, w)).astype(np.float32) for h, w in [(5, 7), (1, 1), (30, 40), (9, 2)]]
    mixed = sd.vl_hog_render(grids, K, variant)
    for g, got in zip(grids, mixed):
        alone = sd.vl_hog_render(g[None], K, variant)[0]
        assert torch.equal(got, alone)
        assert np.array_equal(got.cpu().numpy(), ref.Hog(variant, K).render(g))
    batch = np.stack([rng.standard_normal((31, 6, 8)).astype(np.float32) for _ in range(3)])
    out = sd.vl_hog_render(batch, K, variant)
    assert out.shape == (3, 6 * 21, 8 * 21)
    for i in range(3):
        assert torch.equal(out[i], sd.vl_hog_render(batch[i:i + 1], K, variant)[0])


@pytest.mark.parametrize("K,variant", [(1, 0), (4, 1), (9, 0), (9, 1), (16, 1)])
def test_relayout_is_numpy_gather(sd, K, variant):
    rng = np.random.default_rng(K * 2 + variant)
    dd = 3 * K + 4 if variant else 4 * K
    perm = sd.vl_hog_permutation(variant, K)
    for h, w in [(1, 1), (5, 33), (135, 240), (40, 7)]:
        f = rng.standard_normal((2, dd, h, w)).astype(np.float32)
        flipped = f[:, perm, :, ::-1]
        assert np.array_equal(_relayout(sd, f, K, variant, 1, 0), flipped)
        assert np.array_equal(sd.vl_hog_flip(f, K, variant).cpu().numpy(), flipped)
        assert np.array_equal(_relayout(sd, f, K, variant, 0, 1), np.swapaxes(f, 2, 3))
        assert np.array_equal(_relayout(sd, f, K, variant, 1, 1), np.swapaxes(flipped, 2, 3))
        twice = sd.vl_hog_flip(sd.vl_hog_flip(f, K, variant), K, variant).cpu().numpy()
        assert np.array_equal(twice.view(np.uint32), f.view(np.uint32))
    mixed = [rng.standard_normal((dd, h, w)).astype(np.float32) for h, w in [(3, 4), (17, 1), (8, 64)]]
    for g, got in zip(mixed, sd.vl_hog_flip(mixed, K, variant)):
        assert np.array_equal(got.cpu().numpy(), g[perm, :, ::-1])


@pytest.mark.parametrize("variant", [0, 1])
def test_flip_is_the_hog_of_the_mirror(sd, variant):
    """HOG(mirror(frame)) ~ flip(HOG(frame)) for frames whose width is a multiple of the cell size (the cell grid is then its
    own mirror image).  Not bit for bit: mirroring reverses the order in which each cell sums its votes, and it negates gx, so
    the float orientation scores gx cos + gy sin of a pixel and of its mirror can round to different bins when the pixel lies
    within float rounding of a bin edge.  Smooth float frames have no exact ties, so only the summation order shows: the
    tolerance is the project's 1e-4 bar, and the worst error is printed."""
    rng = np.random.default_rng(3 + variant)
    worst = 0.0
    for K, cs, (h, w) in [(9, 8, (96, 128)), (4, 11, (55, 55)), (16, 4, (60, 44))]:
        frame = rng.uniform(0, 255, (h, w)).astype(np.float32)
        a = sd.vl_hog(frame[None], cs, K, variant)
        b = sd.vl_hog(np.ascontiguousarray(frame[:, ::-1])[None], cs, K, variant)
        e = rel_err(sd.vl_hog_flip(a, K, variant).cpu().numpy(), b.cpu().numpy())
        worst = max(worst, e)
    print(f"HOG(mirror) vs flip(HOG): worst rel_err {worst:.2e}")
    assert worst <= 1e-4
