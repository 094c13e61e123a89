"""Box scores and the tracking step on frames that keep their channels (sd_hog_box_scores_images, sd_track_faces_images,
sd_track_detect_faces_images, sd_bgr2gray_images and their Python front ends), bit for bit unless stated:
  - one 8-bit channel with nearest bins is hog_box_scores, at the grey test's filter and cell sizes;
  - 8-bit frames of 2, 3, 5 and 16 channels and float frames of 1 and 3, both orientation assignments and both variants: the
    scores are the 3 x 3 maximum of vl_hog_correlate(vl_hog(crop)) of the restated crop (tests/box_crop_images_ref.py), in
    planar, interleaved and strided layouts and at per-frame sizes; many 16-channel float boxes (several slices) equal the same
    boxes scored a few at a time;
  - the grey frames passed as one 8-bit channel give the grey step (track_faces, track_and_detect at track_overlap 0, 0.5, 1);
  - colour and float frames: landmarks are the grey step's on their grey, scores hog_box_scores(multichannel=True)'s of the
    returned boxes, and track_and_detect the composition with vl_hog_detect(multichannel=True);
  - sd_bgr2gray_images gives sd_upload_frames' grey at mixed sizes and in several layouts;
  - a colour FaceTracker on a translated colour video with a colour-trained filter;
  - refused calls write nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import box_crop_images_ref as ref
import synth
import track_detect_ref
from colour_examples import examples_bgr

pytestmark = pytest.mark.gpu

CS, K, FW, FH = 8, 9, 6, 6
SCALES = [2.0 ** (-k / 4) for k in range(2, 14)]
NEG = float("-inf")


def _grey(golden):
    return [golden.examples[f"gray{i}"] for i in range(5)]


def _filter(seed, fw=FW, fh=FH, variant=1):
    dd = 3 * K + 4 if variant == 1 else 4 * K
    rng = np.random.default_rng(seed)
    return torch.from_numpy(rng.normal(0, 0.1, (dd, fh, fw)).astype(np.float32)).cuda(), float(rng.normal(0, 0.5))


def _bits(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def _eq(a, b):
    a, b = _bits(a), _bits(b)
    return a.shape == b.shape and np.array_equal(a, b)


def _boxes(rng, frames, per_frame=4):
    box_frame, boxes = [], []
    for i, fr in enumerate(frames):
        H, W = fr.shape[:2]
        for _ in range(per_frame):
            w, h = int(rng.integers(4, W // 2)), int(rng.integers(4, H // 2))
            for x, y in ((int(rng.integers(0, W - w)), int(rng.integers(0, H - h))), (-w // 2, int(rng.integers(0, H - h))),
                         (W - w // 3, H - h // 2), (-3 * w, -2 * h)):
                box_frame.append(i)
                boxes.append((x, y, w, h))
    return box_frame, boxes


def _max9(scores):
    out = []
    for sc in scores:
        v = sc.reshape(-1).cpu().numpy()
        ok = v[~np.isnan(v)]
        out.append(np.float32(np.nan) if ok.size == 0 else v[int(np.flatnonzero(v == ok.max())[0])])
    return np.array(out, np.float32)


def _composed(sd, oracle, frames, box_frame, boxes, f, b, fw, fh, cs, variant, bil):
    crops = [ref.box_crop(oracle, frames[i], bx, fw, fh, cs) for i, bx in zip(box_frame, boxes)]
    maps = sd.vl_hog(np.stack(crops), cs, K, variant, bilinear_orientations=bil, channels_last=True)
    return _max9(sd.vl_hog_correlate(list(maps), f[None], K, variant, bias=torch.tensor([b])))


@pytest.mark.parametrize("fw,fh,cs", [(6, 6, 8), (1, 1, 4), (32, 32, 2), (32, 3, 4), (5, 9, 6)])
def test_one_grey_channel_is_hog_box_scores(sd, fw, fh, cs):
    frames = [synth.smooth_images(1, 97, 131, seed=21)[0], synth.smooth_images(1, 64, 200, seed=22)[0]]
    box_frame, boxes = _boxes(np.random.default_rng(fw * 7 + fh + cs), frames)
    f, b = _filter(fw + fh, fw, fh)
    want = sd.hog_box_scores(frames, box_frame, boxes, f, b, cs, K)
    assert _eq(sd.hog_box_scores(frames, box_frame, boxes, f, b, cs, K, multichannel=True), want)     # per-frame sizes
    dev = torch.from_numpy(np.stack([frames[0]] * 2)).cuda()
    sel = [k for k, i in enumerate(box_frame) if i == 0]
    bf0 = [k % 2 for k in range(len(sel))]
    want0 = sd.hog_box_scores(dev, bf0, [boxes[k] for k in sel], f, b, cs, K)
    assert _eq(want0, want[sel])
    assert _eq(sd.hog_box_scores(dev, bf0, [boxes[k] for k in sel], f, b, cs, K, multichannel=True), want0)


CASES = [(np.uint8, 2), (np.uint8, 3), (np.uint8, 5), (np.uint8, 16), (np.float32, 1), (np.float32, 3)]


def _colour_frames(dtype, C, seed):
    out = []
    for k, (H, W) in enumerate(((97, 131), (64, 200))):
        g = np.stack([synth.smooth_images(1, H, W, seed=seed + 10 * k + c, sigma=1.0)[0] for c in range(C)], axis=-1)
        out.append(g.astype(np.float32) / np.float32(255) if dtype == np.float32 else g)
    return out


@pytest.mark.parametrize("dtype,C", CASES)
@pytest.mark.parametrize("bil", [False, True])
@pytest.mark.parametrize("variant", [0, 1])
def test_scores_equal_the_composition(sd, oracle, dtype, C, bil, variant):
    fl = dtype == np.float32
    frames = _colour_frames(dtype, C, 3 * C + bil)
    box_frame, boxes = _boxes(np.random.default_rng(C + 10 * variant + 100 * bil), frames, 2)
    # context rectangles of the crop's own size, (FW + 2) CS x (FH + 2) CS: the copy branch, inside and across the frame's edge
    box_frame += [0, 0, 1]
    boxes += [(20, 15, FW * CS, FH * CS), (-10, -3, FW * CS, FH * CS), (150, 20, FW * CS, FH * CS)]
    f, b = _filter(C + variant, variant=variant)
    kw = dict(multichannel=True, bilinear_orientations=bil, float_frames=fl)
    got = sd.hog_box_scores(frames, box_frame, boxes, f, b, CS, K, variant, **kw)          # per-frame sizes, interleaved
    want = _composed(sd, oracle, frames, box_frame, boxes, f, b, FW, FH, CS, variant, bil)
    assert _eq(got, want)
    # one size: interleaved, planar and strided views of the same pixels
    sel = [k for k, i in enumerate(box_frame) if i == 0]
    bf, bx = [0] * len(sel), [boxes[k] for k in sel]
    inter = torch.from_numpy(frames[0][None]).cuda()
    planar = inter.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
    big = torch.zeros((1, 97 + 3, 2 * 131 + 5, C + 2), dtype=inter.dtype, device="cuda")
    big[:, 2:99, 3:3 + 2 * 131:2, 1:C + 1] = inter
    strided = big[:, 2:99, 3:3 + 2 * 131:2, 1:C + 1]
    for t in (inter, planar, strided):
        assert _eq(sd.hog_box_scores(t, bf, bx, f, b, CS, K, variant, **kw), got[sel])


def test_many_float_boxes_equal_few_at_a_time(sd):
    """16 float channels at cs 8 and a 32 x 32 filter: 272 x 272 x 16 floats, 4.7 MB per crop, so 200 boxes take 15 slices of
    64 MB, and 7 boxes one."""
    frames = _colour_frames(np.float32, 16, 77)
    rng = np.random.default_rng(5)
    box_frame, boxes = _boxes(rng, frames, 25)
    f, b = _filter(8, 32, 32)
    kw = dict(multichannel=True, float_frames=True)
    got = sd.hog_box_scores(frames, box_frame, boxes, f, b, CS, K, **kw)
    assert len(boxes) == 200
    parts = [sd.hog_box_scores(frames, box_frame[i:i + 7], boxes[i:i + 7], f, b, CS, K, **kw) for i in range(0, 200, 7)]
    assert _eq(got, torch.cat(parts))


@pytest.fixture(scope="module")
def model(sd, golden):
    m = sd.load_detection_model(golden.model_path)
    x = m.detect_faces(_grey(golden), np.arange(5), boxes=golden.examples["boxes"])
    return m, x


def _prev_rows(x):
    return np.array([0, 1, 2, 3, 4, 2, 0]), np.concatenate([x, x[[2, 0]] + np.float32(3)])


def test_grey_frames_as_one_channel_are_the_grey_step(sd, golden, model):
    m, x = model
    frames = torch.from_numpy(synth.smooth_images(3, 360, 480, seed=9)).cuda()
    grey = _grey(golden)
    face, prev = _prev_rows(x)
    filt = _filter(3)
    a = m.track_faces(grey, face, prev, filt, (FW, FH), CS, K, 0.0)
    c = m.track_faces(grey, face, prev, filt, (FW, FH), CS, K, 0.0, multichannel=True)   # a list: per-frame tables
    for g, w in zip(c, a):
        assert _eq(g, w)
    boxes = synth.face_boxes(3, 360, 480, seed=9)
    p = m.detect_faces(list(frames.cpu().numpy()), np.arange(3), boxes=boxes)
    a = m.track_faces(frames, [0, 1, 2, 2], p[[0, 1, 2, 2]], filt, (FW, FH), CS, K, 0.0)
    c = m.track_faces(frames, [0, 1, 2, 2], p[[0, 1, 2, 2]], filt, (FW, FH), CS, K, 0.0, multichannel=True)    # read in place
    for g, w in zip(c, a):
        assert _eq(g, w)
    wide = torch.zeros((3, 360, 480, 3), dtype=torch.uint8, device="cuda")
    wide[..., 1] = frames
    c = m.track_faces(wide[..., 1:2], [0, 1, 2, 2], p[[0, 1, 2, 2]], filt, (FW, FH), CS, K, 0.0, multichannel=True)   # strided grey
    for g, w in zip(c, a):
        assert _eq(g, w)
    frames5 = grey + list(synth.smooth_images(2, 480, 640, seed=42))
    face5 = np.concatenate([face, [5, 6]])
    prev5 = np.concatenate([prev, np.stack([sd.align_mean(m.get_mean(), (100, 80, 150, 150)), sd.align_mean(m.get_mean(), (210, 120, 130, 130))])])
    for t_ov in (0.0, 0.5, 1.0):
        args = (frames5, face5, prev5, filt, (FW, FH), CS, K, 0.0, SCALES, [1, 5, 6], NEG)
        a = m.track_and_detect(*args, track_overlap=t_ov, max_detections=4)
        c = m.track_and_detect(*args, track_overlap=t_ov, max_detections=4, multichannel=True)
        for g, w in zip(c, a):
            assert _eq(g, w) if isinstance(w, torch.Tensor) else g == w, t_ov


def _compose_detect(sd, m, frames, grey, face, prev, filt, thr, listed, det_thr, t_ov, kw, max_det=4):
    """track_and_detect on colour or float frames composed from the calls it is made of (kw: the frames' options)."""
    P = 2 * m.num_landmarks
    old = m.track_faces(frames, face, prev, filt, (FW, FH), CS, K, thr, grey_frames=kw.get("grey_frames"),
                        **{k: v for k, v in kw.items() if k != "grey_frames"})
    old = [t.cpu().numpy() for t in old]
    opts = {k: v for k, v in kw.items() if k != "grey_frames"}
    d = sd.vl_hog_detect([frames[i] for i in listed], SCALES, filt[0][None], CS, K, det_thr, bias=torch.tensor([filt[1]]),
                         max_detections=max_det, **opts)
    det_frame, det_boxes = np.asarray(listed, np.int32)[d.frame], d.boxes
    keep = track_detect_ref.associate(det_frame, det_boxes, face, old[1], old[3], t_ov)
    nf, nb = det_frame[keep], det_boxes[keep]
    n = len(nf)
    lm = m.detect_faces(grey, nf, boxes=nb) if n else np.zeros((0, P), np.float32)
    B, valid = (t.cpu().numpy() for t in sd.track_boxes(lm, m)) if n else (np.zeros((0, 4), np.int32), np.zeros(0, bool))
    sc = np.full(n, np.nan, np.float32)
    if valid.any():
        sc[valid] = sd.hog_box_scores(frames, nf[valid], B[valid], filt[0], filt[1], CS, K, **opts).cpu().numpy()
    alive3 = np.concatenate([old[3], valid & (sc > np.float32(thr))])
    frame = np.concatenate([face, nf]).astype(np.int32)
    boxes = np.concatenate([old[1], B]).astype(np.int32)
    scores = np.concatenate([old[2], sc]).astype(np.float32)
    alive = track_detect_ref.merge(frame, boxes, scores, alive3, len(face), t_ov)
    return np.concatenate([old[0], lm]).astype(np.float32), boxes, scores, alive, frame, n


@pytest.mark.parametrize("kind", ["colour", "colour_bilinear", "float", "float_bilinear"])
def test_colour_and_float_frames(sd, golden, model, kind):
    m, x = model
    grey = _grey(golden)
    colour = examples_bgr(golden)
    bil = kind.endswith("bilinear")
    if kind.startswith("float"):
        frames = [c.astype(np.float32) / np.float32(255) for c in colour]
        kw = dict(multichannel=True, bilinear_orientations=bil, float_frames=True, grey_frames=grey)
    else:
        frames = colour
        kw = dict(multichannel=True, bilinear_orientations=bil)
    opts = {k: v for k, v in kw.items() if k != "grey_frames"}
    face, prev = _prev_rows(x)
    filt = _filter(11)
    out = m.track_faces(frames, face, prev, filt, (FW, FH), CS, K, 0.0, **kw)
    want = m.track_faces(grey, face, prev, filt, (FW, FH), CS, K, 0.0)
    assert _eq(out.landmarks, want.landmarks) and _eq(out.boxes, want.boxes)
    assert _eq(out.scores, sd.hog_box_scores(frames, face, out.boxes, filt[0], filt[1], CS, K, **opts))
    assert _eq(out.alive, out.scores.cpu().numpy() > 0)
    for t_ov in (0.0, 0.5, 1.0):
        got = m.track_and_detect(frames, face, prev, filt, (FW, FH), CS, K, 0.0, SCALES, [1, 3], NEG, track_overlap=t_ov,
                                 max_detections=4, **kw)
        comp = _compose_detect(sd, m, frames, grey, face, prev, filt, 0.0, [1, 3], NEG, t_ov, kw)
        for name, g, w in zip(("landmarks", "boxes", "scores", "alive", "frame", "num_new"), got, comp):
            assert (_eq(g, w) if isinstance(g, torch.Tensor) else g == w), (t_ov, name)


def test_bgr2gray_images_is_the_upload_grey(sd, golden):
    lib, ctx = sd._capi.lib(), sd.default_context()
    grey = _grey(golden)
    colour = examples_bgr(golden)

    def convert(hi):
        n = C.c_size_t(0)
        assert lib.sd_bgr2gray_images(ctx.h, C.byref(hi), None, C.byref(n), None) == 0
        buf = torch.full((n.value,), 7, dtype=torch.uint8, device="cuda")
        ib = sd.ImageBatchC()
        assert lib.sd_bgr2gray_images(ctx.h, C.byref(hi), sd._capi.ptr(buf), C.byref(n), C.byref(ib)) == 0
        return buf, ib

    def frames_of(buf, ib, sizes):
        b = buf.cpu().numpy()
        if not ib.d_frames:
            p = ib.row_stride
            return [b[i * ib.image_stride:(i + 1) * ib.image_stride].reshape(ib.height, p)[:, :ib.width] for i in range(ib.count)]
        table = np.frombuffer(b[ib.d_frames - buf.data_ptr():].tobytes()[:24 * len(sizes)], dtype=np.int32).reshape(-1, 6)
        out = []
        for (h, w), row in zip(sizes, table):
            off = int(row[4]) | (int(row[5]) << 32)
            out.append(b[off:off + h * row[2]].reshape(h, row[2])[:, :w])
        return out

    # mixed sizes, interleaved, packed by the front end; against sd_upload_frames of the same host frames
    keep, hi, sizes = sd._hog_images(colour, True, ctx, lambda w, h: None)
    buf, ib = convert(hi)
    recs, arrays = sd._host_frames(colour)
    up, uib = sd._upload_host_frames(recs, ctx)
    assert buf.numel() == up.numel() and bool(ib.d_frames) and bool(uib.d_frames)
    for g, u, w in zip(frames_of(buf, ib, sizes), frames_of(up, uib, sizes), grey):
        assert np.array_equal(g, u) and np.array_equal(g, w)
    # one size: interleaved, planar and strided batches
    c0 = torch.from_numpy(np.stack([colour[2], colour[2][::-1].copy()])).cuda()
    want = [grey[2], grey[2][::-1]]
    big = torch.zeros((2, c0.shape[1] + 1, 2 * c0.shape[2], 5), dtype=torch.uint8, device="cuda")
    big[:, 1:, ::2, 1:4] = c0
    for t in (c0, c0.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1), big[:, 1:, ::2, 1:4]):
        keep, hi, sizes = sd._hog_images(t, True, ctx, lambda w, h: None)
        buf, ib = convert(hi)
        assert not ib.d_frames and ib.row_stride % 16 == 0
        for g, w in zip(frames_of(buf, ib, sizes), want):
            assert np.array_equal(g, w)


def _translate(frame, tx, ty):
    out = np.zeros_like(frame)
    H, W = frame.shape[:2]
    out[max(ty, 0):H + min(ty, 0), max(tx, 0):W + min(tx, 0)] = frame[max(-ty, 0):H - max(ty, 0), max(-tx, 0):W - max(tx, 0)]
    return out


def test_colour_face_tracker_on_a_translated_video(sd, golden, oracle, model):
    """The five colour example faces translated 3 px right and 2 px up per step, tracked by a colour FaceTracker with a filter
    trained on the colour frames: every face stays tracked within the grey scenario's bound on detect's error, ids stay put, and
    noise frames in two extra streams never start a track."""
    m, x = model
    om = oracle.Model(golden.model_path)
    colour = examples_bgr(golden)
    boxes = golden.examples["boxes"]
    hf = sd.train_hog_filter(colour, np.arange(5), boxes, SCALES, (FW, FH), CS, K, flip_positives=True, multichannel=True)
    ids_l = [int(s) - 1 for s in m.landmark_ids]
    gt_rows = np.stack([np.concatenate([golden.examples[f"pts{i}"][ids_l, 0], golden.examples[f"pts{i}"][ids_l, 1]]) for i in range(5)])
    noise_rgb = lambda k, seed: [np.ascontiguousarray(np.repeat(n[..., None], 3, axis=2)) for n in synth.smooth_images(k, 480, 640, seed=seed)]
    filt = (hf.filter, hf.bias)
    # the threshold: between the faces' scores along the video and the best rows the detector starts on noise
    r = m.track_and_detect(noise_rgb(4, 300), [], np.zeros((0, 44), np.float32), filt, (FW, FH), CS, K, NEG, SCALES, range(4), NEG,
                           track_overlap=1.0, max_detections=16, multichannel=True)
    noise_max = float(np.nanmax(r.scores.cpu().numpy()))
    xs, face_min = x, np.inf
    for step in range(1, 9):
        out = m.track_faces([_translate(c, 3 * step, -2 * step) for c in colour], np.arange(5), xs, filt, (FW, FH), CS, K, NEG,
                            multichannel=True)
        xs, face_min = out.landmarks.cpu().numpy(), min(face_min, float(out.scores.min()))
    print(f"noise rows <= {noise_max:.3f}, faces >= {face_min:.3f}")
    assert face_min > noise_max
    thr = (face_min + noise_max) / 2
    tr = sd.FaceTracker(m, filt, (FW, FH), CS, K, thr, SCALES, thr, multichannel=True)
    tr.landmarks = torch.from_numpy(x).cuda()
    tr.frame = torch.arange(5, dtype=torch.int32, device="cuda")
    tr.ids = torch.arange(5, device="cuda")
    tr.next_id = 5
    for step in range(1, 9):
        tx, ty = 3 * step, -2 * step
        frames = [_translate(c, tx, ty) for c in colour] + noise_rgb(2, 400 + step)
        ids, frame, lm, _ = tr.step(frames)
        ids, frame, lm = ids.cpu().numpy(), frame.cpu().numpy(), lm.cpu().numpy()
        assert frame.tolist() == [0, 1, 2, 3, 4] and ids.tolist() == [0, 1, 2, 3, 4], step     # stable ids, no track on noise
        gt = (gt_rows + np.concatenate([np.full(22, tx), np.full(22, ty)])).astype(np.float32)
        err = sd.calculate_normalised_landmark_errors(lm, gt, m.landmark_ids, om.right_ids, om.left_ids).cpu().numpy().mean(1)
        d = m.detect_faces([_translate(g, tx, ty) for g in _grey(golden)], np.arange(5), boxes=boxes + np.array([tx, ty, 0, 0]))
        ref_err = sd.calculate_normalised_landmark_errors(d, gt, m.landmark_ids, om.right_ids, om.left_ids).cpu().numpy().mean(1)
        assert (err <= ref_err + 0.03).all(), (step, err, ref_err)


def test_refusals_write_nothing(sd, golden, model):
    m, x = model
    lib, ctx, ptr = sd._capi.lib(), m.ctx, sd._capi.ptr
    grey = torch.from_numpy(synth.smooth_images(2, 240, 320, seed=5)).cuda()
    ib = sd.ImageBatchC(C.c_void_p(grey.data_ptr()), 320, 240, 320, 240 * 320, 2)
    colour = torch.from_numpy(np.repeat(synth.smooth_images(2, 240, 320, seed=5)[..., None], 3, axis=3)).cuda()
    fl = torch.zeros((2 * 240 * 320 * 3 + 1,), dtype=torch.float32, device="cuda")

    def images(t=colour, dtype=0, channels=3, count=2, w=320, h=240, data=None):
        hi = sd.HogImagesC()
        hi.d_data = data if data is not None else t.data_ptr()
        hi.dtype, hi.channels, hi.count = dtype, channels, count
        hi.frame = sd.HogImageC(w, h, 0, 3 * w, 3, 1)
        hi.image_stride = 3 * w * h
        hi.d_frames = None
        return hi

    prev = torch.from_numpy(np.stack([sd.align_mean(m.get_mean(), (60, 40, 120, 120))] * 3)).cuda()
    idx = torch.tensor([0, 1, 1], dtype=torch.int32, device="cuda")
    f, b = _filter(3)
    P = 2 * m.num_landmarks

    def outs():
        return (torch.full((3, P), -5.0, device="cuda"), torch.full((3, 4), -5, dtype=torch.int32, device="cuda"),
                torch.full((3,), -5.0, device="cuda"), torch.full((3,), 77, dtype=torch.uint8, device="cuda"))

    def track(hi, bil=0):
        o = outs()
        rc = lib.sd_track_faces_images(ctx.h, m._m, C.byref(ib), C.byref(hi), bil, ptr(idx), ptr(prev), 3, ptr(f), FW, FH, C.c_float(b),
                                       CS, K, 1, C.c_float(0.0), *(ptr(t) for t in o))
        return rc, o

    def written(o):
        return not all(bool((t == v).all()) for t, v in zip(o, (-5.0, -5, -5.0, 77)))

    assert track(images())[0] == 0
    unaligned = images(dtype=1, data=fl.data_ptr() + 2)
    for rc, o in (track(images(count=1)), track(images(w=319)), track(images(h=241)), track(images(dtype=2)),
                  track(images(channels=0)), track(images(channels=17)), track(images(), bil=2), track(unaligned)):
        assert rc == 1 and not written(o)
    scales = np.asarray(SCALES, np.float64)
    param = sd._capi.TrackDetectParamC(scales.ctypes.data_as(C.c_void_p), len(SCALES), 0, 0, 0.0, 0.5, 0.5, 64, 4)
    listed = np.array([0], np.int32)
    R = 3 + 4
    o = (torch.full((R, P), -5.0, device="cuda"), torch.full((R, 4), -5, dtype=torch.int32, device="cuda"),
         torch.full((R,), -5.0, device="cuda"), torch.full((R,), 77, dtype=torch.uint8, device="cuda"),
         torch.full((R,), -5, dtype=torch.int32, device="cuda"))
    n = C.c_int32(-9)
    rc = lib.sd_track_detect_faces_images(ctx.h, m._m, C.byref(ib), C.byref(images(w=321)), 0, ptr(idx), ptr(prev), 3, ptr(f), FW, FH,
                                          C.c_float(b), CS, K, 1, C.c_float(0.0), listed.ctypes.data_as(C.c_void_p), 1, C.byref(param),
                                          *(ptr(t) for t in o), C.byref(n))
    assert rc == 1 and n.value == -9 and not written(o[:4]) and bool((o[4] == -5).all())
    sc = torch.full((2,), -5.0, device="cuda")
    bf = torch.tensor([0, 1], dtype=torch.int32, device="cuda")
    bx = torch.tensor([[10, 10, 40, 40], [300, 200, 50, 50]], dtype=torch.int32, device="cuda")
    for hi, bil in ((images(dtype=2), 0), (images(channels=17), 0), (images(), 2), (unaligned, 0)):
        rc = lib.sd_hog_box_scores_images(ctx.h, C.byref(hi), bil, ptr(bf), ptr(bx), 2, ptr(f), FW, FH, C.c_float(b), CS, K, 1, ptr(sc))
        assert rc == 1 and bool((sc == -5.0).all())
    assert lib.sd_sync(ctx.h) == 0
    fframes = [c.astype(np.float32) for c in examples_bgr(golden)]
    with pytest.raises(ValueError):
        m.track_faces(fframes, [0], x[:1], (f, b), (FW, FH), CS, K, 0.0, multichannel=True, float_frames=True)   # no grey_frames
    with pytest.raises(ValueError):
        sd.hog_box_scores(fframes, [0], [(10, 10, 40, 40)], f, b, CS, K, multichannel=True)                     # float needs float_frames
