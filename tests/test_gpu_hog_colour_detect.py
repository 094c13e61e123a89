"""Detection and training on colour HOG (multichannel=True of train_hog_filter, vl_hog_detect and vl_hog_part_detect).

- On one channel the colour trainer is the grey trainer bit for bit (filter, bias, every round's counts and solve, negative
  cache); on three identical channels colour detect and part detect are grey detect and part detect.
- Objects that differ from their background only in chroma (frames whose grey conversion is flat) have no grey HOG at all; a
  filter trained on the colour features finds every held-out object as its frame's top detection.
- On the colour golden examples a colour filter finds each face, and its boxes chain into detect_faces."""
import numpy as np
import pytest
import torch

import hog_train_ref as T
from colour_examples import bgr_with_gray, examples_bgr

pytestmark = pytest.mark.gpu

CELL, K, SIDE = 8, 9, 6
COUNTS = [f for f in T.COUNTS]


def _same_filter(a, b):
    assert torch.equal(a.filter.view(torch.int32), b.filter.view(torch.int32)) and np.float32(a.bias) == np.float32(b.bias)
    assert np.array_equal(a.negatives, b.negatives)
    assert [{k: r[k] for k in COUNTS + ["solve"]} for r in a.report] == [{k: r[k] for k in COUNTS + ["solve"]} for r in b.report]


def test_one_channel_trainer_is_the_grey_trainer(sd):
    frames, boxes = T.planted_frames(21, 8, 240, 180, sides=(48, 96))
    frames = list(frames[:6]) + [f[:150, :200] for f in frames[6:]]          # two sizes: a descriptor table
    scales = T.detector_scales(240, 180, CELL, SIDE)
    kw = dict(lam=0.01, rounds=2, negatives_per_frame=16, max_negatives=300, flip_positives=True)
    grey = sd.train_hog_filter(frames, np.arange(8), boxes, scales, (SIDE, SIDE), CELL, K, **kw)
    colour = sd.train_hog_filter(frames, np.arange(8), boxes, scales, (SIDE, SIDE), CELL, K, multichannel=True, **kw)
    _same_filter(colour, grey)
    batch = torch.from_numpy(np.stack(frames[:6])).cuda()
    _same_filter(sd.train_hog_filter(batch, np.arange(6), boxes[:6], scales, (SIDE, SIDE), CELL, K, multichannel=True, **kw),
                 sd.train_hog_filter(batch, np.arange(6), boxes[:6], scales, (SIDE, SIDE), CELL, K, **kw))


def test_identical_channels_detect_as_grey(sd):
    rng = np.random.default_rng(3)
    frames, _ = T.planted_frames(22, 4, 200, 150, sides=(40, 80))
    grey = list(frames[:3]) + [frames[3][:97, :131]]
    three = [np.ascontiguousarray(np.stack([g] * 3, -1)) for g in grey]
    dd = 3 * K + 4
    filters = rng.normal(0, 0.2, (2, dd, 4, 5)).astype(np.float32)
    scales = [1.0, 0.8, 0.5]
    a = sd.vl_hog_detect(grey, scales, filters, CELL, K, threshold=-1.0, bias=[0.1, -0.2], pad=(1, 2), max_detections=40)
    b = sd.vl_hog_detect(three, scales, filters, CELL, K, threshold=-1.0, bias=[0.1, -0.2], pad=(1, 2), max_detections=40,
                         multichannel=True)
    assert len(a.frame) > 0
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))
    Q, P = 2, 3
    model = sd.HogPartModel(filters[:, :, :3, :4], [0.0, 0.3], rng.normal(0, 0.2, (Q, P, dd, 2, 3)).astype(np.float32),
                            rng.integers(0, 5, (Q, P, 2)), np.tile([0.05, 0.0, 0.05, 0.0], (Q, P, 1)), (1, 0), (0, 1), 3)
    a = sd.vl_hog_part_detect(grey, [1.0, 0.5], model, CELL, K, threshold=-2.0, max_detections=30)
    b = sd.vl_hog_part_detect(three, [1.0, 0.5], model, CELL, K, threshold=-2.0, max_detections=30, multichannel=True)
    assert len(a.frame) > 0
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def _chroma_frames(seed, n, w, h):
    """Frames of flat grey 128 whose objects and distractors live only in B and R (bgr_with_gray keeps BGR2GRAY at 128)."""
    pattern, boxes = T.planted_frames(seed, n, w, h, sides=(48, 64))
    out = []
    for p in pattern:
        d = (p.astype(np.int64) - 128) // 2
        out.append(bgr_with_gray(np.full((h, w), 128, np.uint8), d, -d))
    return out, boxes


def test_chroma_only_objects(sd, oracle):
    frames, boxes = _chroma_frames(41, 28, 200, 150)
    for f in frames[:4]:
        assert np.array_equal(oracle.bgr2gray_u8(f), np.full(f.shape[:2], 128, np.uint8))
    scales = T.detector_scales(200, 150, CELL, SIDE)
    # the grey route sees nothing: every cell of every level has the features of the flat background
    feats, _ = sd.vl_hog_pyramid(frames[:4], scales, CELL, K)
    for row in feats:
        for t in row:
            if t is not None:
                assert torch.equal(t, t[:, :1, :1].expand_as(t))
    train, test = np.arange(24), np.arange(24, 28)
    hf = sd.train_hog_filter([frames[i] for i in train], np.arange(24), boxes[train], scales, (SIDE, SIDE), CELL, K, lam=0.01,
                             rounds=3, negatives_per_frame=16, max_negatives=4000, flip_positives=True, multichannel=True)
    d = sd.vl_hog_detect([frames[i] for i in test], scales, hf.filter[None], CELL, K, threshold=-10.0, bias=[hf.bias], overlap=0.3,
                         max_detections=4, multichannel=True)
    for j, i in enumerate(test):
        k = int(np.flatnonzero(d.frame == j)[0])
        iou = _iou(d.boxes[k], boxes[i])
        print(f"held-out frame {i}: top {d.boxes[k].tolist()} score {d.scores[k]:.3f}, object {boxes[i].tolist()}, IoU {iou:.3f}")
        assert iou >= 0.5


def _iou(a, b):
    x, y, w, h = (int(v) for v in a)
    bx, by, bw, bh = (int(v) for v in b)
    iw = max(0, min(x + w, bx + bw) - max(x, bx))
    ih = max(0, min(y + h, by + bh) - max(y, by))
    return iw * ih / (w * h + bw * bh - iw * ih)


def test_golden_colour_faces_train_and_chain_to_landmarks(sd, golden):
    frames = examples_bgr(golden)
    boxes = np.asarray(golden.examples["boxes"][:5], np.int32)
    side = 8
    sides = [int(b[2]) for b in boxes]
    s_hi, s_lo = side * CELL * 1.3 / min(sides), side * CELL * 0.7 / max(sides)
    scales = [s_hi * (s_lo / s_hi) ** (k / 11) for k in range(12)]
    hf = sd.train_hog_filter(frames, np.arange(5), boxes, scales, (side, side), CELL, K, lam=0.01, flip_positives=True, rounds=3,
                             negatives_per_frame=64, max_negatives=4000, multichannel=True)
    d = sd.vl_hog_detect(frames, scales, hf.filter[None], CELL, K, threshold=-10.0, bias=[hf.bias], overlap=0.3, max_detections=8,
                         multichannel=True)
    model = sd.load_detection_model(golden.model_path)
    for i in range(5):
        k = int(np.flatnonzero(d.frame == i)[0])
        iou = _iou(d.boxes[k], boxes[i])
        print(f"face {i}: top detection {d.boxes[k].tolist()} score {d.scores[k]:.3f}, golden {boxes[i].tolist()}, IoU {iou:.3f}")
        assert iou >= 0.5
        lm = model.detect_faces([frames[i]], np.zeros(1, np.int32), boxes=d.boxes[k:k + 1])
        assert np.isfinite(lm).all()
