"""The tracking step with the detector inside it (sd_track_detect_faces, detection_model.track_and_detect, FaceTracker) against
the calls it is made of and the association and merge restatement of tests/track_detect_ref.py, bit for bit unless stated:
  - with no frame listed and track_overlap 1 the step is track_faces;
  - with no tracks, every frame listed and track_overlap 1 the new rows are vl_hog_detect's detections, their landmarks
    detect_faces' from those boxes, their boxes and scores track_boxes' and hog_box_scores';
  - in general (faces, duplicated tracks, tracks on noise, a listed subset of frames) every output is the composition of
    track_faces, vl_hog_detect, the association, detect_faces, track_boxes, hog_box_scores and the merge;
  - streams split over two calls give the rows of one call, and two runs are identical;
  - FaceTracker on a scenario of golden faces entering, moving through and leaving noise frames;
  - refused calls write nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import synth
import track_detect_ref

pytestmark = pytest.mark.gpu

CS, K, FW, FH = 8, 9, 6, 6
SCALES = [2.0 ** (-k / 4) for k in range(2, 14)]
NEG = float("-inf")


def _grey(golden):
    return [golden.examples[f"gray{i}"] for i in range(5)]


@pytest.fixture(scope="module")
def trained(sd, golden):
    """The rcr_22 model, a face filter trained on the golden frames, and the golden faces' landmarks."""
    m = sd.load_detection_model(golden.model_path)
    grey = _grey(golden)
    hf = sd.train_hog_filter(grey, np.arange(5), golden.examples["boxes"], SCALES, (FW, FH), CS, K, flip_positives=True)
    x = m.detect_faces(grey, np.arange(5), boxes=golden.examples["boxes"])
    return m, (hf.filter, hf.bias), x


def _random_filter(seed):
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.normal(0, 0.1, (3 * K + 4, FH, FW)).astype(np.float32)).cuda(), float(rng.normal(0, 0.5))


def _step(m, frames, face, prev, filt, thr, listed, det_thr, t_ov, max_det=4):
    return m.track_and_detect(frames, face, prev, filt, (FW, FH), CS, K, thr, SCALES, listed, det_thr, track_overlap=t_ov,
                              max_detections=max_det)


def _np(step):
    return [t.cpu().numpy() if isinstance(t, torch.Tensor) else t for t in step]


def _equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def _compose(sd, m, frames, face, prev, filt, thr, listed, det_thr, t_ov, max_det=4):
    """The step composed from today's calls and the restatement: (landmarks, boxes, scores, alive, frame, num_new) on the host."""
    P = 2 * m.num_landmarks
    prev = np.asarray(prev, np.float32).reshape(-1, P)
    face = np.asarray(face, np.int32)
    T = len(face)
    if T:
        old = _np(m.track_faces(frames, face, prev, filt, (FW, FH), CS, K, thr))
    else:
        old = [np.zeros((0, P), np.float32), np.zeros((0, 4), np.int32), np.zeros(0, np.float32), np.zeros(0, bool)]
    f = torch.as_tensor(filt[0]).reshape(1, -1, FH, FW)
    det_frame, det_boxes = np.zeros(0, np.int32), np.zeros((0, 4), np.int32)
    if len(listed):
        d = sd.vl_hog_detect([frames[i] for i in listed], SCALES, f, CS, K, det_thr, bias=torch.tensor([filt[1]], dtype=torch.float32),
                             max_detections=max_det)
        det_frame, det_boxes = np.asarray(listed, np.int32)[d.frame], d.boxes
    keep = track_detect_ref.associate(det_frame, det_boxes, face, old[1], old[3], t_ov)
    nf, nb = det_frame[keep], det_boxes[keep]
    n = len(nf)
    lm = m.detect_faces(frames, nf, boxes=nb) if n else np.zeros((0, P), np.float32)
    B, valid = (t.cpu().numpy() for t in sd.track_boxes(lm, m)) if n else (np.zeros((0, 4), np.int32), np.zeros(0, bool))
    sc = np.full(n, np.nan, np.float32)
    if valid.any():
        sc[valid] = sd.hog_box_scores(frames, nf[valid], B[valid], filt[0], filt[1], CS, K).cpu().numpy()
    alive3 = np.concatenate([old[3], valid & (sc > np.float32(thr))])
    frame = np.concatenate([face, nf]).astype(np.int32)
    boxes = np.concatenate([old[1], B]).astype(np.int32)
    scores = np.concatenate([old[2], sc]).astype(np.float32)
    alive = track_detect_ref.merge(frame, boxes, scores, alive3, T, t_ov)
    return np.concatenate([old[0], lm]).astype(np.float32), boxes, scores, alive, frame, n


def _check(got, want):
    names = ("landmarks", "boxes", "scores", "alive", "frame", "num_new")
    for name, g, w in zip(names, _np(got), want):
        assert _equal(g, w), name


def test_no_listed_frame_is_track_faces(sd, golden, trained):
    m, _, x = trained
    grey = _grey(golden)
    filt = _random_filter(3)
    face = np.array([0, 1, 2, 3, 4, 2, 0])
    prev = np.concatenate([x, x[[2, 0]] + np.float32(3)])
    tf = _np(m.track_faces(grey, face, prev, filt, (FW, FH), CS, K, 0.0))
    got = _np(_step(m, grey, face, prev, filt, 0.0, [], NEG, 1.0))
    for g, w in zip(got[:4], tf):
        assert _equal(g, w)
    assert _equal(got[4], face) and got[5] == 0


def test_no_tracks_every_frame_listed_is_detect(sd, golden, trained):
    m, filt, _ = trained
    frames = _grey(golden) + list(synth.smooth_images(2, 360, 480, seed=41))
    listed = list(range(len(frames)))
    got = _np(_step(m, frames, [], np.zeros((0, 44), np.float32), filt, 0.0, listed, NEG, 1.0))
    d = sd.vl_hog_detect(frames, SCALES, filt[0][None], CS, K, NEG, bias=torch.tensor([filt[1]]), max_detections=4)
    assert got[5] == len(d.frame) == 4 * len(frames)
    assert _equal(got[4], d.frame)
    want_lm = m.detect_faces(frames, d.frame, boxes=d.boxes)
    assert _equal(got[0], want_lm)
    B, valid = sd.track_boxes(want_lm, m)
    assert _equal(got[1], B.cpu().numpy())
    assert valid.all()
    assert _equal(got[2], sd.hog_box_scores(frames, d.frame, B, filt[0], filt[1], CS, K).cpu().numpy())
    assert _equal(got[3], got[2] > 0)
    _check(got, _compose(sd, m, frames, [], np.zeros((0, 44)), filt, 0.0, listed, NEG, 1.0))


def _general(golden, x, m, sd):
    frames = _grey(golden) + list(synth.smooth_images(3, 480, 640, seed=42))
    box = lambda x0, y0, s: sd.align_mean(m.get_mean(), (x0, y0, s, s))
    face = np.array([0, 1, 2, 3, 4, 0, 2, 5, 6, 6, 3])
    prev = np.concatenate([x, x[[0]], x[[2]] + np.float32(1.5), np.stack([box(100, 80, 150), box(200, 120, 130), box(210, 120, 130)]),
                           x[[3]] - np.float32(40)]).astype(np.float32)
    return frames, face, prev, [6, 1, 5, 3, 7]


@pytest.mark.parametrize("t_ov", [0.5, 0.0, 1.0])
def test_general_step_equals_the_composition(sd, golden, trained, t_ov):
    m, filt, x = trained
    frames, face, prev, listed = _general(golden, x, m, sd)
    thr = float(np.nanmedian(m.track_faces(frames, face, prev, filt, (FW, FH), CS, K, 0.0).scores.cpu().numpy()))
    got = _step(m, frames, face, prev, filt, thr, listed, thr - 0.5, t_ov)
    want = _compose(sd, m, frames, face, prev, filt, thr, listed, thr - 0.5, t_ov)
    print(f"t_ov {t_ov}: threshold {thr:.3f}, {want[5]} new rows, alive {want[3].astype(int)}")
    _check(got, want)
    # a device batch of equal frames
    dev = torch.from_numpy(np.stack([np.pad(f, ((0, 1024 - f.shape[0]), (0, 728 - f.shape[1]))) for f in frames[:5]])).cuda()
    got_dev = _step(m, dev, face[:5], prev[:5], filt, thr, [4, 0], thr - 0.5, t_ov)
    want_dev = _compose(sd, m, list(dev.cpu().numpy()), face[:5], prev[:5], filt, thr, [4, 0], thr - 0.5, t_ov)
    _check(got_dev, want_dev)


def test_streams_split_over_calls_and_runs_repeat(sd, golden, trained):
    m, filt, x = trained
    frames, face, prev, listed = _general(golden, x, m, sd)
    thr = 0.0
    one = _np(_step(m, frames, face, prev, filt, thr, listed, -0.5, 0.5))
    again = _np(_step(m, frames, face, prev, filt, thr, listed, -0.5, 0.5))
    for a, b in zip(one, again):
        assert _equal(a, b)
    # streams 0..3 and 4..7 in two calls; the tracks of each half in their original order
    A, B = face < 4, face >= 4
    ra = _np(_step(m, frames[:4], face[A], prev[A], filt, thr, [f for f in listed if f < 4], -0.5, 0.5))
    rb = _np(_step(m, frames[4:], face[B] - 4, prev[B], filt, thr, [f - 4 for f in listed if f >= 4], -0.5, 0.5))
    T, Ta, Tb = len(face), int(A.sum()), int(B.sum())
    order = np.concatenate([np.flatnonzero(A), np.flatnonzero(B)])
    # the one call's new rows: listed order [6, 1, 5, 3, 7] -> frames of each half in the same relative order
    new_frame = one[4][T:]
    for k in range(4):
        old_split = np.concatenate([ra[k][:Ta], rb[k][:Tb]])
        assert _equal(one[k][:T][order], old_split), k
        new_a = one[k][T:][new_frame < 4]
        new_b = one[k][T:][new_frame >= 4]
        assert _equal(new_a, ra[k][Ta:]) and _equal(new_b, rb[k][Tb:]), k
    assert one[5] == ra[5] + rb[5]


def _paste(canvas, face, x, y):
    out = canvas.copy()
    h, w = face.shape
    out[y:y + h, x:x + w] = face
    return out


def test_face_tracker_scenario(sd, golden, oracle, trained):
    """Three streams of 480 x 640 noise: golden face 0 enters stream 0 at step 1 and leaves at step 7, face 1 enters stream 1 at
    step 3 and stays, stream 2 never shows a face; faces move 3 px right and 2 px down per step."""
    m, filt, _ = trained
    om = oracle.Model(golden.model_path)
    grey = _grey(golden)
    boxes = golden.examples["boxes"]
    ids_l = [int(s) - 1 for s in m.landmark_ids]
    crops, gts = [], []
    for i in (0, 1):
        bx, by, bw, bh = (int(v) for v in boxes[i])
        e = bw // 4
        x0, y0 = max(bx - e, 0), max(by - e, 0)
        crops.append(grey[i][y0:by + bh + e, x0:bx + bw + e])
        pts = golden.examples[f"pts{i}"]
        gts.append((np.concatenate([pts[ids_l, 0] - x0, pts[ids_l, 1] - y0]).astype(np.float32), (bx - x0, by - y0, bw, bh)))
    present = {0: range(1, 7), 1: range(3, 10)}
    origin = {0: (40, 30), 1: (300, 120)}

    def scene(step, seed):
        noise = list(synth.smooth_images(3, 480, 640, seed=seed))
        where = {}
        for s in (0, 1):
            if step in present[s]:
                x, y = origin[s][0] + 3 * step, origin[s][1] + 2 * step
                noise[s] = _paste(noise[s], crops[s], x, y)
                where[s] = (x, y)
        return noise, where

    # threshold: between the detector's best new rows on noise and the scores of tracked faces
    calib = list(synth.smooth_images(8, 480, 640, seed=500))
    r = m.track_and_detect(calib, [], np.zeros((0, 44), np.float32), filt, (FW, FH), CS, K, NEG, SCALES, range(8), NEG,
                           track_overlap=1.0, max_detections=16)
    noise_max = float(np.nanmax(r.scores.cpu().numpy()))
    face_scores = []
    for step in range(1, 7):
        fr, where = scene(step, 1000 + step)
        for s in (0, 1):
            if s in where:
                gt_box = np.array(gts[s][1]) + np.array([where[s][0], where[s][1], 0, 0])
                lm = m.detect_faces(fr, [s], boxes=gt_box[None])
                B, _ = sd.track_boxes(lm, m)
                face_scores.append(float(sd.hog_box_scores(fr, [s], B, filt[0], filt[1], CS, K).cpu().numpy()[0]))
    print(f"noise new rows <= {noise_max:.3f}, tracked faces >= {min(face_scores):.3f}")
    assert min(face_scores) > noise_max
    thr = (min(face_scores) + noise_max) / 2

    tr = sd.FaceTracker(m, filt, (FW, FH), CS, K, thr, SCALES, thr)
    track_id = {}
    for step in range(10):
        fr, where = scene(step, 1000 + step)
        ids, frame, lm, _ = tr.step(fr)
        ids, frame, lm = ids.cpu().numpy(), frame.cpu().numpy(), lm.cpu().numpy()
        assert not (frame == 2).any(), step                                   # noise never starts a track
        for s in (0, 1):
            rows = np.flatnonzero(frame == s)
            if step in present[s] and step > present[s][0]:
                assert len(rows) == 1, (step, s, rows)                       # one track within one step of entering
                track_id.setdefault(s, ids[rows[0]])
                assert ids[rows[0]] == track_id[s], step                     # a stable id
                if step >= present[s][0] + 2:
                    x, y = where[s]
                    gt = gts[s][0] + np.concatenate([np.full(22, x), np.full(22, y)]).astype(np.float32)
                    gt_box = np.array(gts[s][1]) + np.array([x, y, 0, 0])
                    d = m.detect_faces(fr, [s], boxes=gt_box[None])
                    err = sd.calculate_normalised_landmark_errors(lm[rows], np.stack([gt]), m.landmark_ids, om.right_ids,
                                                                  om.left_ids).cpu().numpy().mean()
                    ref = sd.calculate_normalised_landmark_errors(d, np.stack([gt]), m.landmark_ids, om.right_ids,
                                                                  om.left_ids).cpu().numpy().mean()
                    assert err <= ref + 0.03, (step, s, err, ref)
            elif step not in present[s]:
                assert len(rows) == 0, (step, s)                             # a face that left ends its track
    # a second track on face 1 (a copy: equal scores, so the row order decides): the two merge into the older id
    s1 = int(np.flatnonzero(tr.frame.cpu().numpy() == 1)[0])
    tr.ids = torch.cat([tr.ids, torch.tensor([tr.next_id], device=tr.ids.device)])
    tr.frame = torch.cat([tr.frame, tr.frame[s1:s1 + 1]])
    tr.landmarks = torch.cat([tr.landmarks, tr.landmarks[s1:s1 + 1]])
    tr.next_id += 1
    fr, _ = scene(9, 1009)
    ids, frame, _, _ = tr.step(fr)
    sel = frame.cpu().numpy() == 1
    assert sel.sum() == 1 and ids.cpu().numpy()[sel][0] == track_id[1]


def test_refusals_write_nothing(sd, golden, trained):
    m, filt, x = trained
    lib, ctx = sd._capi.lib(), m.ctx
    frames = torch.from_numpy(synth.smooth_images(2, 240, 320, seed=5)).cuda()
    ib = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), 320, 240, 320, 240 * 320, 2)
    prev = torch.from_numpy(np.stack([sd.align_mean(m.get_mean(), (60, 40, 120, 120))] * 3)).cuda()
    f, b = filt
    P = 2 * m.num_landmarks
    R = 3 + 2 * 4

    def call(idx=(0, 1, 1), listed=(1, 0), fw=FW, fh=FH, cs=CS, k=K, thr=0.0, **kw):
        p = dict(scales=SCALES, pad=(0, 0), det=-1.0, nms=0.5, tov=0.5, mc=4096, md=4)
        p.update(kw)
        sc = np.ascontiguousarray(p["scales"], np.float64)
        par = sd._capi.TrackDetectParamC(sc.ctypes.data_as(C.c_void_p), sc.size, p["pad"][0], p["pad"][1], p["det"], p["nms"],
                                         p["tov"], p["mc"], p["md"])
        o = (torch.full((R, P), -5.0, device="cuda"), torch.full((R, 4), -5, dtype=torch.int32, device="cuda"),
             torch.full((R,), -5.0, device="cuda"), torch.full((R,), 77, dtype=torch.uint8, device="cuda"),
             torch.full((R,), -5, dtype=torch.int32, device="cuda"))
        lst = np.ascontiguousarray(listed, np.int32)
        n = C.c_int32(-7)
        d_idx = torch.tensor(idx, dtype=torch.int32, device="cuda")
        rc = lib.sd_track_detect_faces(ctx.h, m._m, C.byref(ib), sd._capi.ptr(d_idx), sd._capi.ptr(prev), 3, sd._capi.ptr(f), fw, fh,
                                       C.c_float(b), cs, k, 1, C.c_float(thr), lst.ctypes.data_as(C.c_void_p), lst.size, C.byref(par),
                                       *(sd._capi.ptr(t) for t in o), C.byref(n))
        untouched = all(bool((t == v).all()) for t, v in zip(o, (-5.0, -5, -5.0, 77, -5))) and n.value == -7
        return rc, untouched

    assert call()[0] == 0
    cases = [dict(listed=(2,)), dict(listed=(-1,)), dict(listed=(1, 1)), dict(tov=1.5), dict(tov=-0.1), dict(nms=1.01),
             dict(thr=float("nan")), dict(det=float("nan")), dict(md=0), dict(md=9, mc=8), dict(mc=8193), dict(scales=[0.5, 0.0]),
             dict(scales=[5.0]), dict(scales=[]), dict(pad=(FW, 0)), dict(pad=(0, -1)), dict(fw=33), dict(cs=0), dict(k=17),
             dict(idx=(0, 2, 1))]
    for kw in cases:
        rc, untouched = call(**kw)
        assert rc == 1 and untouched, kw
    assert lib.sd_sync(ctx.h) == 0
    with pytest.raises(sd.SdError):
        m.track_and_detect(frames, [0], prev[:1], filt, (FW, FH), CS, K, 0.0, SCALES, [0, 0], 0.0)
