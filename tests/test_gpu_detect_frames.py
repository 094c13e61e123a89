"""detect on host frames of any size, grey or colour, several faces per frame (sd_detect_faces_host / sd_detect_faces_device)."""
import ctypes as C

import numpy as np
import pytest
import torch

import synth
from colour_examples import examples_bgr
from test_gpu_detect import _rounding_margin

pytestmark = pytest.mark.gpu

SIZES = [(240, 320), (200, 264), (300, 416)]


def _pinned(frame, pad=16):
    """A pinned copy of `frame` whose rows are 16-byte aligned and `pad` bytes longer than the pixels (a CPU tensor view)."""
    h, w = frame.shape[:2]
    ch = 1 if frame.ndim == 2 else frame.shape[2]
    pitch = (w * ch + 15) // 16 * 16 + pad
    buf = torch.zeros((h, pitch), dtype=torch.uint8).pin_memory()
    buf[:, :w * ch] = torch.from_numpy(np.ascontiguousarray(frame).reshape(h, w * ch))
    return buf[:, :w * ch].view(h, w, 3) if ch == 3 else buf[:, :w]


def _colour(h, w, seed):
    return np.ascontiguousarray(np.stack([synth.smooth_images(1, h, w, seed=seed + c)[0] for c in range(3)], axis=-1))


@pytest.fixture(scope="module")
def model(sd, golden):
    return sd.load_detection_model(golden.model_path)


@pytest.fixture(scope="module")
def scene():
    """Colour frames of three sizes, 0 to 4 faces each (one frame has none), about 25 % of the boxes over the border, faces
    listed in shuffled frame order."""
    rng = np.random.default_rng(2024)
    frames, face_frame, boxes = [], [], []
    counts = [2, 0, 4, 1, 3, 2, 1, 4, 3]
    for f, n in enumerate(counts):
        h, w = SIZES[f % 3]
        frames.append(_colour(h, w, seed=100 + 7 * f))
        for b in synth.face_boxes(n, h, w, seed=500 + f, border_fraction=0.25):
            face_frame.append(f)
            boxes.append(b)
    perm = rng.permutation(len(face_frame))
    return frames, np.array(face_frame, dtype=np.int32)[perm], np.array(boxes, dtype=np.int32)[perm]


def test_reference_photos_in_one_call(sd, model, golden):
    """The reference's five example frames in colour (five sizes) in one call: the reference landmarks to 1e-4, bit-identical to
    detect() on each grey frame, from pageable arrays (whole-frame route) and from pinned padded rows (ROI route)."""
    frames = examples_bgr(golden)
    boxes = golden.examples["boxes"]
    ctx = model.ctx
    l0 = ctx.launches()
    full = model.detect_faces(frames, np.arange(5), boxes=boxes)
    l1 = ctx.launches()
    fb0 = ctx.roi_fallbacks()
    roi = model.detect_faces([_pinned(f) for f in frames], np.arange(5), boxes=boxes)
    l2, fb = ctx.launches(), ctx.roi_fallbacks() - fb0
    print("launches: whole frames", l1 - l0, "ROI", l2 - l1, "ROI fallbacks", fb)
    if fb == 0:
        assert l2 - l1 < l1 - l0          # one gather launch instead of one colour conversion per frame
    assert np.array_equal(roi, full)
    for i in range(5):
        ref = golden.detect[f"landmarks{i}"]
        assert np.max(np.abs(full[i] - ref)) <= 1e-4 * np.max(np.abs(ref)), i
        assert np.array_equal(full[i], model.detect(golden.examples[f"gray{i}"], boxes[i])), i


def test_several_faces_per_colour_frame(sd, oracle, golden, model, scene):
    frames, face_frame, boxes = scene
    got = model.detect_faces(frames, face_frame, boxes=boxes)
    # pinned frames (ROI route) give the same landmarks
    assert np.array_equal(model.detect_faces([_pinned(f) for f in frames], face_frame, boxes=boxes), got)
    gray = [oracle.bgr2gray_u8(f) for f in frames]
    x0 = np.stack([sd.align_mean(model.get_mean(), b) for b in boxes]).astype(np.float32)
    om = oracle.Model(golden.model_path)
    for size in SIZES:
        fids = [f for f in range(len(frames)) if frames[f].shape[:2] == size]
        faces = np.array([i for i in range(len(face_frame)) if face_frame[i] in fids])
        # the frames duplicated once per face through the device-resident batch
        dup = torch.from_numpy(np.stack([gray[face_frame[i]] for i in faces])).cuda()
        dev = model.detect_batch_device(dup, torch.from_numpy(x0[faces]).cuda()).cpu().numpy()
        assert np.array_equal(dev, got[faces]), size
        # each frame resident once, faces indexed into it (sd_detect_faces_device)
        resident = sd.bgr2gray(np.stack([frames[f] for f in fids]))
        index = np.array([fids.index(face_frame[i]) for i in faces], dtype=np.int32)
        idx = model.detect_batch_device(resident, torch.from_numpy(x0[faces]).cuda(), image_index=index).cpu().numpy()
        assert np.array_equal(idx, got[faces]), size
        # the oracle, face by face: 1e-4, except a face proven to sit on a rounding tie (see test_gpu_detect)
        ref = om.detect_batch(np.stack([gray[face_frame[i]] for i in faces]), boxes[faces], threads=8)
        per_face = np.max(np.abs(got[faces] - ref), axis=1) / np.max(np.abs(ref))
        for j in np.nonzero(per_face > 1e-4)[0]:
            near = _rounding_margin(oracle, om, gray[face_frame[faces[j]]], x0[faces[j]])
            print(f"size {size} face {faces[j]}: rel err {per_face[j]:.2e}, rounding margin {near:.2e}")
            assert near <= 5e-5
        assert np.max(np.abs(got[faces] - ref)) <= 1.0


def test_tracking_from_initialisations(sd, oracle, golden, model, scene):
    frames, face_frame, boxes = scene
    x0 = np.stack([sd.align_mean(model.get_mean(), b) for b in boxes]).astype(np.float32)
    first = model.detect_faces(frames, face_frame, boxes=boxes)
    assert np.array_equal(model.detect_faces(frames, face_frame, initialisations=x0), first)
    # a second pass from the first pass's landmarks (the next video frame), against the oracle's detect(image, initialisation)
    second = model.detect_faces([_pinned(f) for f in frames], face_frame, initialisations=first)
    assert np.array_equal(second, model.detect_faces(frames, face_frame, initialisations=first))
    om = oracle.Model(golden.model_path)
    for i in range(len(face_frame)):
        gray = oracle.bgr2gray_u8(frames[face_frame[i]])
        ref = om.detect_init(gray, first[i])
        err = np.max(np.abs(second[i] - ref)) / np.max(np.abs(ref))
        if err > 1e-4:
            near = _rounding_margin(oracle, om, gray, first[i])
            print(f"face {i}: rel err {err:.2e}, rounding margin {near:.2e}")
            assert near <= 5e-5
            assert np.max(np.abs(second[i] - ref)) <= 1.0


def test_invalid_inputs_raise_and_leave_the_output(sd, model, golden):
    from superviseddescent_b200 import _capi
    lib = _capi.lib()
    gray = np.ascontiguousarray(golden.examples["gray1"])
    h, w = gray.shape
    box = np.ascontiguousarray(golden.examples["boxes"][1:2], dtype=np.int32)
    x0 = sd.align_mean(model.get_mean(), box[0]).reshape(1, -1)
    P = 2 * model.num_landmarks

    def call(frame, idx, boxes, init):
        frames = (_capi.HostFrameC * 1)(frame)
        out = np.full((1, P), 7.0, dtype=np.float32)
        i = np.array([idx], dtype=np.int32)
        rc = lib.sd_detect_faces_host(model.ctx.h, model._m, frames, 1, i.ctypes.data_as(C.c_void_p), 1,
                                      None if boxes is None else boxes.ctypes.data_as(C.c_void_p),
                                      None if init is None else init.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        return rc, out

    good = _capi.HostFrameC(gray.ctypes.data, w, h, w, 1)
    assert call(good, 0, box, None)[0] == 0
    cases = {
        "index past the end": (good, 1, box, None),
        "negative index": (good, -1, box, None),
        "two channels": (_capi.HostFrameC(gray.ctypes.data, w // 2, h, w, 2), 0, box, None),
        "both boxes and initialisations": (good, 0, box, x0),
        "neither boxes nor initialisations": (good, 0, None, None),
        "row_stride < width * channels": (_capi.HostFrameC(gray.ctypes.data, w // 3 + 1, h, w - 1, 3), 0, box, None),
    }
    for name, args in cases.items():
        rc, out = call(*args)
        assert rc == 1, name                                  # SD_ERR_INVALID
        assert np.all(out == 7.0), name
    with pytest.raises(sd.SdError):
        model.detect_faces([np.zeros((40, 40, 4), dtype=np.uint8)], [0], boxes=[[0, 0, 30, 30]])
    with pytest.raises(sd.SdError):                           # degenerate face: a zero-sized box
        model.detect_faces([gray], [0], boxes=[[100, 100, 0, 0]])
    assert model.detect_faces([gray], np.zeros(0, dtype=np.int32), boxes=np.zeros((0, 4), dtype=np.int32)).shape == (0, P)
    assert np.array_equal(model.detect_faces([gray], [0], boxes=box)[0], model.detect(gray, box[0]))   # the context still works
