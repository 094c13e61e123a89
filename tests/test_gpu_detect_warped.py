"""Detect on warped faces (sd_detect_faces_device_warped through detection_model.detect_faces(warps=...) and
detect_batch_device(warps=...)) against detect on the materialised virtual frames (cv2.warpAffine of the grey frame,
WARP_INVERSE_MAP), bit for bit; identity warps equal plain detect."""
import cv2
import numpy as np
import pytest
import torch

import sample_warp_ref as SW
import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def faces(sd, golden):
    m = sd.load_detection_model(golden.model_path)
    grey = list(synth.smooth_images(3, 240, 320, seed=21))
    colour = [np.ascontiguousarray(np.stack([g, np.roll(g, 3, 1), np.roll(g, 5, 0)], -1)) for g in grey]
    boxes = synth.face_boxes(6, 240, 320, seed=21)
    face_frame = np.array([0, 1, 2, 0, 1, 2], dtype=np.int32)
    rng = np.random.default_rng(8)
    warps = np.stack([sd.rotation_warp((b[0] + b[2] / 2, b[1] + b[3] / 2), float(rng.uniform(-50, 50)), float(rng.uniform(0.8, 1.2)))
                      for b in boxes])
    sizes = np.array([(320, 240), (300, 260), (320, 240), (200, 180), (320, 240), (360, 250)])
    return m, grey, colour, boxes, face_frame, warps, sizes


def test_detect_faces_warped_equals_materialised(sd, faces):
    m, grey, colour, boxes, ff, warps, sizes = faces
    for frames in (grey, colour):
        g = [f if f.ndim == 2 else cv2.cvtColor(f, cv2.COLOR_BGR2GRAY) for f in frames]
        vs = [SW.materialise(g[f], M, s) for f, M, s in zip(ff, warps, sizes)]
        got = m.detect_faces(frames, ff, boxes=boxes, warps=warps, warp_sizes=sizes)
        want = m.detect_faces(vs, np.arange(len(vs)), boxes=boxes)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        x0 = np.stack([sd.align_mean(m.get_mean(), b) for b in boxes]) + np.float32(0.75)
        got = m.detect_faces(frames, ff, initialisations=x0, warps=warps, warp_sizes=sizes)
        want = m.detect_faces(vs, np.arange(len(vs)), initialisations=x0)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_detect_batch_device_warped_equals_materialised(sd, faces):
    m, grey, _, boxes, ff, warps, _ = faces
    images = torch.from_numpy(np.stack(grey)).cuda()
    x0 = torch.from_numpy(np.stack([sd.align_mean(m.get_mean(), b) for b in boxes])).cuda()
    got = m.detect_batch_device(images, x0, image_index=ff, warps=warps).cpu().numpy()
    vs = torch.from_numpy(np.stack([SW.materialise(grey[f], M, (320, 240)) for f, M in zip(ff, warps)])).cuda()
    want = m.detect_batch_device(vs, x0).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    ident = np.broadcast_to(np.eye(2, 3), (len(ff), 2, 3))
    got = m.detect_batch_device(images, x0, image_index=ff, warps=ident).cpu().numpy()
    want = m.detect_batch_device(images, x0, image_index=ff).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(m.detect_faces(grey, ff, boxes=boxes, warps=ident).view(np.uint32),
                          m.detect_faces(grey, ff, boxes=boxes).view(np.uint32))


def test_detect_warped_refusals(sd, faces):
    m, grey, _, boxes, ff, warps, _ = faces
    images = torch.from_numpy(np.stack(grey)).cuda()
    x0 = torch.from_numpy(np.stack([sd.align_mean(m.get_mean(), b) for b in boxes])).cuda()
    bad = warps.copy()
    bad[2, 0, 0] = np.nan
    with pytest.raises(sd.SdError, match="invalid sample warp"):
        m.detect_batch_device(images, x0, image_index=ff, warps=bad)
    with pytest.raises(sd.SdError, match="out of range"):
        m.detect_batch_device(images, x0, image_index=np.array(ff) | (1 << 30), warps=warps)
    with pytest.raises(ValueError):
        m.detect_batch_device(images, x0, image_index=ff, warps=warps[:2])
    sd.default_context().sync()
