"""One tracking step on the device (sd_track_boxes, sd_hog_box_scores, sd_track_faces) against the numpy restatements of
tests/track_ref.py and the calls it is made of, bit for bit unless stated:
  - the boxes of seeded landmarks equal track_ref's, and the device align_mean equals sd_align_mean (a model whose regressors
    are zero returns its initialisation);
  - a step's landmarks are detect_faces' from the rule-1 boxes on grey and colour host frames, device frames and frames of
    mixed sizes;
  - hog_box_scores is the 3 x 3 maximum of vl_hog_correlate(hog_dense(crop)) of the restated crop, at filter sides 1 and 32;
  - on a video of the golden frames translated a few pixels per step, every track stays alive within a margin of detect's error,
    and smooth-noise frames score below every face and end their tracks;
  - collapsed landmarks and faces too small for a patch end their own tracks only; refused calls write nothing."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import synth
import track_ref
from colour_examples import examples_bgr

pytestmark = pytest.mark.gpu

CS, K, FW, FH = 8, 9, 6, 6
SCALES = [2.0 ** (-k / 4) for k in range(2, 14)]


def _model(sd, golden):
    return sd.load_detection_model(golden.model_path)


def _frames(golden):
    return [golden.examples[f"gray{i}"] for i in range(5)]


def _prev(sd, golden, m):
    """Landmarks to track from: detect on the golden frames from their boxes."""
    return m.detect_faces(_frames(golden), np.arange(5), boxes=golden.examples["boxes"])


def _filter(seed, fw=FW, fh=FH, variant=1):
    dd = 3 * K + 4 if variant == 1 else 4 * K
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.normal(0, 0.1, (dd, fh, fw)).astype(np.float32)).cuda(), float(rng.normal(0, 0.5))


def test_track_boxes_match_the_restatement(sd, golden):
    m = _model(sd, golden)
    mean = m.get_mean()
    rng = np.random.default_rng(1)
    rows = [sd.align_mean(mean, (int(rng.integers(-300, 1500)), int(rng.integers(-300, 900)), int(s), int(s)))
            + rng.normal(0, float(rng.choice([0.0, 0.3, 3.0])), 2 * m.num_landmarks).astype(np.float32)
            for s in rng.integers(8, 600, 500)]
    rows += [np.full(2 * m.num_landmarks, 7.0, np.float32), np.full(2 * m.num_landmarks, np.nan, np.float32),
             np.where(np.arange(2 * m.num_landmarks) == 3, np.float32(np.inf), np.float32(1)).astype(np.float32),
             (mean * np.float32(3e9)).astype(np.float32), (mean * np.float32(0.4)).astype(np.float32)]
    X = np.stack(rows).astype(np.float32)
    boxes, valid = sd.track_boxes(X, m)
    want_b, want_v = track_ref.track_boxes(X, mean)
    assert np.array_equal(valid.cpu().numpy(), want_v)
    assert np.array_equal(boxes.cpu().numpy(), want_b)
    assert want_v[:500].all() and not want_v[500:].any()


def test_device_align_mean_equals_sd_align_mean(sd, golden, oracle):
    """A one-level model with zero regressors returns its initialisation: the step's landmarks are the device align_mean."""
    m = _model(sd, golden)
    om = oracle.Model(golden.model_path)
    hp = m.hog_param(0)
    D, P = m.weights(0).shape
    reg = types.SimpleNamespace(x=torch.zeros((D, P)), regulariser=sd.Regulariser())
    z = sd.detection_model.from_parts(types.SimpleNamespace(regressors=[reg]), m.get_mean(), m.landmark_ids, [hp], om.right_ids,
                                      om.left_ids)
    frames = synth.smooth_images(3, 480, 640, seed=3)
    rng = np.random.default_rng(2)
    boxes = np.array([(int(rng.integers(0, 400)), int(rng.integers(0, 250)), int(s), int(s)) for s in rng.integers(60, 220, 96)])
    prev = np.stack([sd.align_mean(m.get_mean(), b) for b in boxes]).astype(np.float32)
    face = np.arange(96) % 3
    f, b = _filter(4)
    out = z.track_faces(torch.from_numpy(frames).cuda(), face, prev, (f, b), (FW, FH), CS, K, -1e30)
    assert np.array_equal(out.landmarks.cpu().numpy(), prev)
    assert np.array_equal(out.boxes.cpu().numpy(), boxes)


def _check_step(sd, m, frames, face, prev, host_frames):
    f, b = _filter(7)
    out = m.track_faces(frames, face, prev, (f, b), (FW, FH), CS, K, -1e30)
    B, valid = track_ref.track_boxes(prev, m.get_mean())
    assert valid.all()
    want = m.detect_faces(host_frames, face, boxes=B)
    assert np.array_equal(out.landmarks.cpu().numpy(), want)
    B2, valid2 = track_ref.track_boxes(want, m.get_mean())
    assert np.array_equal(out.boxes.cpu().numpy(), B2)
    assert out.alive.cpu().numpy().all()
    return out


def test_step_equals_detect_from_the_rule_boxes(sd, golden):
    m = _model(sd, golden)
    grey = _frames(golden)
    prev = _prev(sd, golden, m)
    face = np.array([0, 1, 2, 3, 4, 2, 0])
    prev = np.concatenate([prev, prev[[2, 0]] + np.float32(4)])
    _check_step(sd, m, grey, face, prev, grey)                                  # grey host frames of mixed sizes
    colour = examples_bgr(golden)
    _check_step(sd, m, colour, face, prev, colour)                              # colour host frames
    _check_step(sd, m, [grey[0], colour[1], grey[2], colour[3], grey[4]], face, prev, grey)   # a mixed table
    dev = synth.smooth_images(4, 240, 320, seed=11)
    boxes = synth.face_boxes(4, 240, 320, seed=11)
    p = m.detect_faces(list(dev), np.arange(4), boxes=boxes)
    _check_step(sd, m, torch.from_numpy(dev).cuda(), np.array([0, 1, 2, 3, 3, 1]), p[[0, 1, 2, 3, 3, 1]], list(dev))


def _restated_scores(sd, oracle, frames, box_frame, boxes, f, b, fw, fh, cs):
    crops = [track_ref.box_crop(oracle, frames[i], bx, fw, fh, cs) for i, bx in zip(box_frame, boxes)]
    maps = sd.hog_dense(np.stack(crops), cs, K)
    s = sd.vl_hog_correlate(list(maps), f[None], K, bias=torch.tensor([b]))
    out = []
    for sc in s:
        v = sc.reshape(-1).cpu().numpy()
        ok = v[~np.isnan(v)]
        out.append(np.float32(np.nan) if ok.size == 0 else v[int(np.flatnonzero(v == ok.max())[0])])
    return np.array(out, np.float32)


@pytest.mark.parametrize("fw,fh,cs", [(6, 6, 8), (1, 1, 4), (32, 32, 2), (32, 3, 4), (5, 9, 6)])
def test_box_scores_equal_the_composition(sd, oracle, fw, fh, cs):
    frames = [synth.smooth_images(1, 97, 131, seed=21)[0], synth.smooth_images(1, 64, 200, seed=22)[0]]
    rng = np.random.default_rng(fw * 7 + fh + cs)
    box_frame, boxes = [], []
    for i, fr in enumerate(frames):
        H, W = fr.shape
        for _ in range(6):
            w, h = int(rng.integers(4, W // 2)), int(rng.integers(4, H // 2))
            for x, y in ((int(rng.integers(0, W - w)), int(rng.integers(0, H - h))), (-w // 2, int(rng.integers(0, H - h))),
                         (W - w // 3, H - h // 2), (-3 * w, -2 * h), (W + 5, 3)):
                box_frame.append(i)
                boxes.append((x, y, w, h))
    f, b = _filter(fw + fh, fw, fh)
    got = sd.hog_box_scores(frames, box_frame, boxes, f, b, cs, K).cpu().numpy()
    want = _restated_scores(sd, oracle, frames, box_frame, boxes, f, b, fw, fh, cs)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the same boxes in one device batch of equal frames: the same scores
    dev = torch.from_numpy(np.stack([frames[0], frames[0]])).cuda()
    sel = [k for k, i in enumerate(box_frame) if i == 0]
    got0 = sd.hog_box_scores(dev, [k % 2 for k in range(len(sel))], [boxes[k] for k in sel], f, b, cs, K).cpu().numpy()
    assert np.array_equal(got0.view(np.uint32), got[sel].view(np.uint32))


def _translate(frame, tx, ty):
    out = np.zeros_like(frame)
    H, W = frame.shape
    out[max(ty, 0):H + min(ty, 0), max(tx, 0):W + min(tx, 0)] = frame[max(-ty, 0):H - max(ty, 0), max(-tx, 0):W - max(tx, 0)]
    return out


def test_tracking_a_translated_video(sd, golden, oracle):
    m = _model(sd, golden)
    om = oracle.Model(golden.model_path)
    grey = _frames(golden)
    boxes = golden.examples["boxes"]
    hf = sd.train_hog_filter(grey, np.arange(5), boxes, SCALES, (FW, FH), CS, K, flip_positives=True)
    gt_rows = np.stack([np.concatenate([golden.examples[f"pts{i}"][[int(s) - 1 for s in m.landmark_ids], 0],
                                        golden.examples[f"pts{i}"][[int(s) - 1 for s in m.landmark_ids], 1]]) for i in range(5)])
    x = m.detect_faces(grey, np.arange(5), boxes=boxes)
    face_scores, noise_scores = [], []
    for step in range(1, 11):
        tx, ty = 3 * step, -2 * step
        frames = [_translate(g, tx, ty) for g in grey]
        gt = (gt_rows + np.concatenate([np.full(22, tx), np.full(22, ty)])).astype(np.float32)
        out = m.track_faces(frames, np.arange(5), x, hf, (FW, FH), CS, K, -1e30)
        assert out.alive.cpu().numpy().all(), step
        x = out.landmarks.cpu().numpy()
        err = sd.calculate_normalised_landmark_errors(x, gt, m.landmark_ids, om.right_ids, om.left_ids).cpu().numpy().mean(1)
        shifted = boxes + np.array([tx, ty, 0, 0])
        d = m.detect_faces(frames, np.arange(5), boxes=shifted)
        ref = sd.calculate_normalised_landmark_errors(d, gt, m.landmark_ids, om.right_ids, om.left_ids).cpu().numpy().mean(1)
        print(f"step {step}: tracked error {np.round(err, 4)}, detect from the box {np.round(ref, 4)}")
        assert (err <= ref + 0.03).all(), (step, err, ref)
        face_scores.append(out.scores.cpu().numpy())
        noise = list(synth.smooth_images(5, 480, 640, seed=100 + step))
        noise_scores.append(sd.hog_box_scores(noise, np.arange(5), out.boxes, hf.filter, hf.bias, CS, K).cpu().numpy())
    face_scores, noise_scores = np.concatenate(face_scores), np.concatenate(noise_scores)
    print(f"face scores >= {face_scores.min():.3f}, noise scores <= {noise_scores.max():.3f}")
    assert face_scores.min() > noise_scores.max()
    threshold = float((face_scores.min() + noise_scores.max()) / 2)
    frames = [_translate(g, 33, -22) for g in grey]                         # step 11
    alive = m.track_faces(frames, np.arange(5), x, hf, (FW, FH), CS, K, threshold).alive.cpu().numpy()
    assert alive.all()
    noise = list(synth.smooth_images(5, 1100, 800, seed=99))
    alive = m.track_faces(noise, np.arange(5), x, hf, (FW, FH), CS, K, threshold).alive.cpu().numpy()
    assert not alive.any()


def test_dying_tracks_leave_the_others_alone(sd, golden):
    m = _model(sd, golden)
    grey = _frames(golden)
    prev = _prev(sd, golden, m)
    f, b = _filter(9)
    base = m.track_faces(grey, np.arange(5), prev, (f, b), (FW, FH), CS, K, -1e30)
    collapsed = np.full(2 * m.num_landmarks, 100.0, np.float32)
    tiny = sd.align_mean(m.get_mean(), (150, 150, 3, 3))
    X = np.stack([collapsed, prev[0], prev[1], tiny, prev[2], prev[3], prev[4], collapsed])
    face = np.array([0, 0, 1, 2, 2, 3, 4, 4])
    out = m.track_faces(grey, face, X, (f, b), (FW, FH), CS, K, -1e30)
    alive = out.alive.cpu().numpy()
    assert alive.tolist() == [False, True, True, False, True, True, True, False]
    lm = out.landmarks.cpu().numpy()
    keep = [1, 2, 4, 5, 6]
    assert np.array_equal(lm[keep], base.landmarks.cpu().numpy())
    assert np.array_equal(out.boxes.cpu().numpy()[keep], base.boxes.cpu().numpy())
    assert np.array_equal(out.scores.cpu().numpy()[keep].view(np.uint32), base.scores.cpu().numpy().view(np.uint32))
    assert np.array_equal(lm[[0, 7]], X[[0, 7]])                                  # a degenerate box keeps prev
    m.ctx.sync()                                                                  # no flag left behind


def test_refusals_write_nothing(sd, golden):
    m = _model(sd, golden)
    lib, ctx = sd._capi.lib(), m.ctx
    frames = torch.from_numpy(synth.smooth_images(2, 240, 320, seed=5)).cuda()
    ib = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), 320, 240, 320, 240 * 320, 2)
    prev = torch.from_numpy(np.stack([sd.align_mean(m.get_mean(), (60, 40, 120, 120))] * 3)).cuda()
    f, b = _filter(3)
    P = 2 * m.num_landmarks

    def outs():
        return (torch.full((3, P), -5.0, device="cuda"), torch.full((3, 4), -5, dtype=torch.int32, device="cuda"),
                torch.full((3,), -5.0, device="cuda"), torch.full((3,), 77, dtype=torch.uint8, device="cuda"))

    def track(idx, fw=FW, fh=FH, cs=CS, k=K, o=None):
        o = o or outs()
        rc = lib.sd_track_faces(ctx.h, m._m, C.byref(ib), sd._capi.ptr(idx), sd._capi.ptr(prev), 3, sd._capi.ptr(f), fw, fh,
                                C.c_float(b), cs, k, 1, C.c_float(0.0), *(sd._capi.ptr(t) for t in o))
        return rc, o

    ok_idx = torch.tensor([0, 1, 1], dtype=torch.int32, device="cuda")
    assert track(ok_idx)[0] == 0
    for rc, o in (track(torch.tensor([0, 2, 1], dtype=torch.int32, device="cuda")), track(ok_idx, fw=33), track(ok_idx, cs=0),
                  track(ok_idx, k=17), track(ok_idx, fw=1, fh=1, cs=1)):
        assert rc == 1
        assert all(bool((t == v).all()) for t, v in zip(o, (-5.0, -5, -5.0, 77)))
    assert lib.sd_sync(ctx.h) == 0                                                 # the refused call left no flag behind

    boxes = torch.tensor([[10, 10, 40, 40], [300, 200, 50, 50]], dtype=torch.int32, device="cuda")
    for bf, bx, fw in ((torch.tensor([0, 2]), boxes, FW), (torch.tensor([0, 1]), boxes * torch.tensor([1, 1, 0, 1], device="cuda"), FW),
                       (torch.tensor([0, 1]), boxes, 0), (torch.tensor([-1, 1]), boxes, FW)):
        sc = torch.full((2,), -5.0, device="cuda")
        rc = lib.sd_hog_box_scores(ctx.h, C.byref(ib), sd._capi.ptr(bf.to("cuda", torch.int32)), sd._capi.ptr(bx.contiguous()), 2,
                                   sd._capi.ptr(f), fw, FH, C.c_float(b), CS, K, 1, sd._capi.ptr(sc))
        assert rc == 1 and bool((sc == -5.0).all())
    # corners inside int32 but a side outside it: x = -2^30, w = 2^30 and fw = 1 make the rectangle 3 * 2^30 px wide
    wide = torch.tensor([[-2 ** 30, 0, 2 ** 30, 10]], dtype=torch.int32, device="cuda")
    sc = torch.full((1,), -5.0, device="cuda")
    rc = lib.sd_hog_box_scores(ctx.h, C.byref(ib), sd._capi.ptr(torch.zeros(1, dtype=torch.int32, device="cuda")), sd._capi.ptr(wide), 1,
                               sd._capi.ptr(f[:, :1, :1].contiguous()), 1, 1, C.c_float(b), CS, K, 1, sd._capi.ptr(sc))
    assert rc == 1 and bool((sc == -5.0).all())
    with pytest.raises(ValueError):
        m.track_faces(frames, [0, 1, 1], prev, (f, b), (FW + 1, FH), CS, K, 0.0)
