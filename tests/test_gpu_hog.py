"""GPU parity of the batched HOG projection (sd_hog_batch) against the CPU oracle, through the C ABI.

Integer results (patch centre, half size, resized 8-bit patch, orientation bin) must be EXACT; the float
descriptors must agree to 1e-4 relative (max-norm / max-abs), the tolerance BASELINE.json states.
"""
import numpy as np
import pytest

import synth
from colour_examples import bgr_with_gray
from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _oracle_params(O, p):
    return O.HogParam(p.variant, p.num_cells, p.cell_size, p.num_bins, p.relative_patch_size)


def _check_level(sd, O, images, x, hog_param, ids, right, left, image_index=None):
    import torch
    ht = sd.HogTransform(images, [hog_param], ids, right, left)
    ridx = [ids.index(s) for s in right]
    lidx = [ids.index(s) for s in left]
    op = _oracle_params(O, hog_param)
    A = ht(x, 0, image_index).cpu().numpy()
    geo, patches, bins = [t.cpu().numpy() for t in ht.debug(x, 0, image_index)]
    fs = hog_param.num_cells * hog_param.cell_size
    worst = 0.0
    for i in range(x.shape[0]):
        img = images[i if image_index is None else image_index[i]]
        cx, cy, half = O.patch_geometry(x[i], op, ridx, lidx)
        assert np.array_equal(geo[i, :, 0], cx) and np.array_equal(geo[i, :, 1], cy) and np.array_equal(geo[i, :, 2], half), f"geometry sample {i}"
        for l in range(len(ids)):
            patch = O.resize_linear_u8(O.crop_patch_u8(img, int(cx[l]), int(cy[l]), int(half[l])), fs, fs)
            assert np.array_equal(patches[i, l], patch), f"resized patch sample {i} landmark {l}"
            ob = O.hog_orientation_bins(patch.astype(np.float32), hog_param.num_bins)
            assert np.array_equal(bins[i, l].astype(np.int32), ob), f"orientation bins sample {i} landmark {l}"
        ref = O.hog_transform(img, x[i], op, ridx, lidx)
        assert A[i, -1] == 1.0
        worst = max(worst, rel_err(A[i], ref))
    assert worst <= TOL, worst
    return worst


def test_hog_rcr22_schedule_on_example_frames(sd, oracle, golden):
    """The shipped rcr_22 schedule (K=4, 5x5 cells of 11/10/8/6 px) on the reference's annotated frames."""
    m = oracle.Model(golden.model_path)
    worst = 0.0
    for i in (0, 2):
        gray = golden.examples[f"gray{i}"]
        x0 = oracle.align_mean(m.mean, golden.examples["boxes"][i]).reshape(1, -1)
        for level in range(4):
            p = m.hog_params[level]
            hp = sd.HoGParam(p.variant, p.num_cells, p.cell_size, p.num_bins, p.relative_patch_size)
            worst = max(worst, _check_level(sd, oracle, gray[None], x0, hp, m.landmark_ids, m.right_ids, m.left_ids))
        feats = sd.HogTransform(gray[None], [sd.HoGParam(1, 5, 11, 4, 1.0)], m.landmark_ids, m.right_ids, m.left_ids)(x0[0], 0)
        assert rel_err(feats.cpu().numpy(), golden.detect[f"features_l0_{i}"]) <= TOL     # committed hog.c golden
    print("hog rcr22 worst rel err", worst)


@pytest.mark.parametrize("K,variant", [(9, 1), (4, 0), (6, 1)])
def test_hog_synthetic_batch_with_border_patches(sd, oracle, golden, K, variant):
    """Seeded synthetic frames, boxes hanging over the border (zero padding), K=9 (31-dim cells),
    Dalal-Triggs, and a generic K that takes the non-templated kernel."""
    m = oracle.Model(golden.model_path)
    images = synth.smooth_images(6, 120, 160, seed=11)
    boxes = synth.face_boxes(6, 120, 160, seed=11, border_fraction=0.5)
    boxes[0] = (-30, -20, 90, 90)
    boxes[1] = (110, 70, 80, 80)
    x = np.stack([oracle.align_mean(m.mean, b) for b in boxes])
    idx = np.array([5, 4, 3, 2, 1, 0], dtype=np.int32)
    for cs, rel in ((11, 1.0), (6, 0.25)):
        hp = sd.HoGParam(variant, 5, cs, K, rel)
        w = _check_level(sd, oracle, images, x, hp, m.landmark_ids, m.right_ids, m.left_ids, image_index=idx)
        print(f"K={K} variant={variant} cs={cs} worst rel err {w:.2e}")


def test_hog_ragged_and_empty_inputs(sd, oracle, golden):
    import torch
    m = oracle.Model(golden.model_path)
    images = synth.smooth_images(2, 64, 64, seed=5)
    ht = sd.HogTransform(images, [sd.HoGParam(1, 5, 6, 4, 0.25)], m.landmark_ids, m.right_ids, m.left_ids)
    empty = torch.empty((0, 44), dtype=torch.float32, device="cuda")
    assert ht(empty, 0).shape == (0, 8801)
    # landmarks far outside the frame -> all-zero patches -> features are exactly the bias-only row
    far = np.full((1, 44), 5000.0, dtype=np.float32)
    far[0, :22] += np.arange(22) * 7
    A = ht(far, 0).cpu().numpy()
    assert A[0, -1] == 1.0 and np.all(A[0, :-1] == 0.0)
    with pytest.raises(RuntimeError):
        sd.HogTransform(images, [sd.HoGParam(1, 5, 6, 4, 0.25)], m.landmark_ids, ["nope"], m.left_ids)(far, 0)


def test_bgr2gray_device_is_bit_exact(sd, oracle, golden):
    """cv::cvtColor(BGR2GRAY) (adaptive_vlhog.hpp:114-120) on the device against the cv2-pinned oracle: the golden crop,
    random frames with widths that exercise the 4-pixel vector path and the scalar tail, and a HogTransform fed with
    colour frames (must equal the one fed with the converted frames)."""
    crop = golden.examples["bgr_crop"]
    got = sd.bgr2gray(crop[None]).cpu().numpy()[0]
    assert np.array_equal(got, golden.examples["bgr_crop_gray"])
    rng = np.random.default_rng(5)
    for (n, h, w) in [(3, 17, 64), (2, 9, 63), (1, 5, 1), (4, 33, 130)]:
        bgr = rng.integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)
        want = np.stack([oracle.bgr2gray_u8(bgr[i]) for i in range(n)])
        assert np.array_equal(sd.bgr2gray(bgr).cpu().numpy(), want), (n, h, w)
    m = oracle.Model(golden.model_path)
    bgr = rng.integers(0, 256, size=(2, 120, 160, 3), dtype=np.uint8)
    gray = np.stack([oracle.bgr2gray_u8(bgr[i]) for i in range(2)])
    x0 = np.stack([oracle.align_mean(m.mean, (30, 20, 90, 90)) for _ in range(2)]).astype(np.float32)
    hp = [sd.HoGParam(1, 5, 11, 4, 1.0)]
    fa = sd.HogTransform(bgr, hp, m.landmark_ids, m.right_ids, m.left_ids)(x0, 0).cpu().numpy()
    fb = sd.HogTransform(gray, hp, m.landmark_ids, m.right_ids, m.left_ids)(x0, 0).cpu().numpy()
    assert np.array_equal(fa, fb)


@pytest.mark.parametrize("variant,nc,cs,K", [(1, 3, 12, 4), (0, 3, 12, 4), (1, 5, 10, 9), (1, 4, 6, 4)])
def test_fixed_patch_hog_transform_vs_oracle(sd, oracle, variant, nc, cs, K):
    """The non-adaptive HogTransform of the reference's hello-world (examples/landmark_detection.cpp:195-261): fixed patch
    of half-size num_cells * (cell_size / 2), zero padding at the border, no resize, no bias.  Landmarks include points
    at and beyond the frame border.  An odd cell size is rejected (the un-resized patch would get a different HOG grid)."""
    import synth
    rng = np.random.default_rng(nc * 100 + cs)
    imgs = synth.smooth_images(3, 120, 160, seed=11)
    L = 7
    x = np.concatenate([rng.uniform(-5, 165, size=(3, L)), rng.uniform(-5, 125, size=(3, L))], axis=1).astype(np.float32)
    x[0, 0], x[0, L] = 0.0, 0.0                                   # patch centred on the corner pixel
    x[1, 1], x[1, L + 1] = 159.5, 119.5                           # cvRound half-to-even at the far corner
    h = sd.FixedHogTransform(imgs, variant, nc, cs, K)
    got = h(x, 0).cpu().numpy()
    hp = oracle.HogParam(variant, nc, cs, K, 0.0)
    want = np.stack([oracle.hog_transform_fixed(imgs[i], x[i], hp) for i in range(3)])
    assert got.shape == want.shape
    err = rel_err(got, want)
    print(f"fixed-patch HOG variant {variant} nc {nc} cs {cs} K {K}: rel err {err:.2e}")
    assert err <= 1e-5
    one = h(x[2], 0, 2).cpu().numpy()                             # predict()'s call shape: one row + image index
    assert np.array_equal(one, got[2])
    with pytest.raises(Exception):
        sd.FixedHogTransform(imgs, variant, nc, 11, K)(x, 0)


def test_hog_frames_of_different_sizes(sd, oracle, golden):
    """The reference's HogTransform takes a std::vector<cv::Mat> of arbitrary sizes (rcr-train reads photographs of different
    resolutions): a list of differently sized frames goes through per-frame descriptors (sd_frame) and must give, frame by
    frame, what the oracle gives -- including patches that hang over each frame's OWN border.  The same frames in B,G,R (one of
    them with a padded row step) must give the same features and debug taps."""
    m = oracle.Model(golden.model_path)
    sizes = [(120, 160), (97, 131), (200, 150), (64, 64)]
    frames = [synth.smooth_images(1, h, w, seed=40 + i)[0] for i, (h, w) in enumerate(sizes)]
    boxes = [(10, 8, 90, 90), (40, 20, 80, 80), (-20, 60, 120, 120), (5, 5, 50, 50)]
    x = np.stack([oracle.align_mean(m.mean, b) for b in boxes]).astype(np.float32)
    rng = np.random.default_rng(41)
    colour = [bgr_with_gray(f, rng.integers(-40, 41, f.shape), rng.integers(-40, 41, f.shape)) for f in frames]
    h1, w1 = sizes[1]
    padded = np.zeros((h1, w1 + 5, 3), dtype=np.uint8)
    padded[:, :w1] = colour[1]
    colour[1] = padded[:, :w1]
    assert all(np.array_equal(oracle.bgr2gray_u8(c), f) for c, f in zip(colour, frames))
    for cs, rel, K in ((11, 1.0, 4), (6, 0.25, 9)):
        hp, ohp = sd.HoGParam(1, 5, cs, K, rel), oracle.HogParam(1, 5, cs, K, rel)
        ht = sd.HogTransform(frames, [hp], m.landmark_ids, m.right_ids, m.left_ids)
        A = ht(x, 0).cpu().numpy()
        geo, patches, bins = ht.debug(x, 0)
        hc = sd.HogTransform(colour, [hp], m.landmark_ids, m.right_ids, m.left_ids)
        assert np.array_equal(hc(x, 0).cpu().numpy(), A), cs
        assert all(np.array_equal(c.cpu().numpy(), g.cpu().numpy()) for c, g in zip(hc.debug(x, 0), (geo, patches, bins))), cs
        for i, f in enumerate(frames):
            ref = oracle.hog_transform(f, x[i], ohp, m.right_idx, m.left_idx)
            assert rel_err(A[i], ref) <= TOL, (i, cs)
            cxs, cys, half = oracle.patch_geometry(x[i], ohp, m.right_idx, m.left_idx)
            for l in range(len(m.landmark_ids)):
                want = oracle.resize_linear_u8(oracle.crop_patch_u8(f, int(cxs[l]), int(cys[l]), int(half[l])), 5 * cs, 5 * cs)
                assert np.array_equal(patches[i, l].cpu().numpy(), want), (i, l, cs)    # integer result: bit exact
    with pytest.raises(ValueError):
        sd.HogTransform([frames[0], np.zeros((3, 4, 5, 6), np.uint8)], [hp], m.landmark_ids, m.right_ids, m.left_ids)
