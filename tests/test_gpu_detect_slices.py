"""detect on host frames (sd_detect_faces_host, csrc/sd_model.cu) where its work is cut up, and the upload the HogTransform
front ends share (sd_upload_frames).

The call takes one of two routes (DESIGN §4.5), and both cut their work into chunks at sizes the other detect tests never
reach:
  whole-frame route  every referenced frame, in upload order (faces stable-sorted by frame), costs H * round16(W) grey bytes
                     plus H * round16(3 W) B,G,R bytes if it is colour; a chunk closes when the next frame would pass 128 MiB.
                     Chunks alternate between two staging buffers; a chunk of equally sized frames is a strided batch, any
                     other chunk a descriptor table.
  ROI route          (every referenced frame pinned, with 16-byte aligned rows) every face, in caller order, costs the bytes
                     of its region of interest (face_roi); a chunk closes when the next face would pass 48 MiB.  A face whose
                     patches leave its ROI is redone on the whole-frame route; an ROI larger than 48 MiB moves the whole call
                     to the whole-frame route.
The chunk rules and face_roi are restated here (face_roi in float32) and checked against the launch counter.  Landmarks are
checked bit for bit against one detect over device-resident frames (detect_batch_device with an image index: no chunks, no
ROI), and a few faces against the oracle to 1e-4.  Translation models (every weight 0 but the bias row) move every face by a
known multiple of its inter-eye distance per level, so which faces leave their ROI is known in closed form.
"""
import functools

import numpy as np
import pytest
import torch

from test_gpu_detect import _rounding_margin
from test_gpu_hog_configs import (FEATURE_TOL, H as KH, W as KW, Layout, _frames, _sample, compare, device_batch, largest_staged,
                                  run_kernel, smem_layout, truth)

MiB = 1 << 20
FULL_CHUNK = 128 * MiB           # detect_faces_full: frame bytes per staging buffer
ROI_CHUNK = 48 * MiB             # detect_faces_roi: packed ROI bytes per staging buffer (SD_STAGE_HALF_BYTES)
UPLOAD_CHUNK = 64 * MiB          # sd_upload_frames: B,G,R scratch per chunk
F32 = np.float32


def _round16(v):
    return (v + 15) // 16 * 16


def _channels(frame):
    return 1 if frame.ndim == 2 else frame.shape[2]


# ---- frames ------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _base():
    """A 2400 x 4400 low-pass noise texture (separable Gaussian, sigma 3) that every frame is cut from."""
    h, w, r, sigma = 2400, 4400, 9, 3.0
    k = np.exp(-0.5 * (np.arange(-r, r + 1) / sigma) ** 2).astype(F32)
    k /= k.sum()
    img = np.random.default_rng(77).random((h + 2 * r, w + 2 * r), dtype=F32)
    a = sum(k[i] * img[i:i + h] for i in range(2 * r + 1))
    b = sum(k[i] * a[:, i:i + w] for i in range(2 * r + 1))
    b = (b - b.min()) / (b.max() - b.min())
    return np.round(b * 255).astype(np.uint8)


def _grey(h, w, seed):
    base = _base()
    if h > base.shape[0] or w > base.shape[1]:
        base = np.tile(base, (-(-h // base.shape[0]), -(-w // base.shape[1])))
    rng = np.random.default_rng(seed)
    y, x = int(rng.integers(0, base.shape[0] - h + 1)), int(rng.integers(0, base.shape[1] - w + 1))
    return np.ascontiguousarray(base[y:y + h, x:x + w])


def _bgr(h, w, seed):
    return np.ascontiguousarray(np.stack([_grey(h, w, seed * 3 + c) for c in range(3)], axis=-1))


class Pinned:
    """Pinned copies of host frames (sd_host_alloc, exact sizes), held until the object goes; counts the bytes it holds."""
    held = 0
    peak = 0

    def __init__(self, sd):
        self.sd, self.bufs, self.bytes = sd, [], 0

    def __call__(self, frame, pitch=None):
        """A pinned copy of `frame` whose rows lie `pitch` bytes apart (default: the row's bytes rounded up to 16)."""
        from superviseddescent_b200 import api
        h, w, ch = frame.shape[0], frame.shape[1], _channels(frame)
        pitch = pitch or _round16(w * ch)
        buf = api._PinnedBuffer(self.sd.default_context(), h * pitch)
        self.bufs.append(buf)
        self.bytes += h * pitch
        Pinned.held += h * pitch
        Pinned.peak = max(Pinned.peak, Pinned.held)
        rows = buf.array.reshape(h, pitch)
        rows[:, :w * ch] = frame.reshape(h, w * ch)
        shape, strides = ((h, w), (pitch, 1)) if ch == 1 else ((h, w, 3), (pitch, 3, 1))
        return np.lib.stride_tricks.as_strided(buf.array, shape=shape, strides=strides)

    def release(self):
        Pinned.held -= self.bytes
        self.bufs, self.bytes = [], 0


# ---- restated rules ----------------------------------------------------------------------------------------------------
def full_bytes(frame):
    h, w = frame.shape[:2]
    return h * _round16(w) + (h * _round16(3 * w) if _channels(frame) == 3 else 0)


def full_chunks(frames, face_frame):
    """detect_faces_full's chunks: lists of frame indices, in upload order."""
    chunks, used = [], 0
    for f in sorted(set(int(i) for i in face_frame)):            # faces stable-sorted by frame: frames in ascending order
        b = full_bytes(frames[f])
        if not chunks or used + b > FULL_CHUNK:
            chunks.append([])
            used = 0
        chunks[-1].append(f)
        used += b
    return chunks


class Geometry:
    """What the restatements need of a model: levels' relative patch sizes, eye indices, HOG parameters (oracle types)."""

    def __init__(self, om):
        self.om = om
        self.rel = [F32(hp.relative_patch_size) for hp in om.hog_params]
        self.right, self.left = list(om.right_idx), list(om.left_idx)


def face_roi(geo, x0, width, height, row_pixels, drift=0.2):
    """face_roi (csrc/sd_model.cu) in float32: (x, y, w, h).  drift: the allowance per inter-eye distance after level 0."""
    x = np.asarray(x0, dtype=F32)
    L = x.size // 2
    minx, maxx, miny, maxy = x[:L].min(), x[:L].max(), x[L:].min(), x[L:].max()

    def mean(idx, off):
        s = F32(0)
        for i in idx:
            s = F32(s + x[i + off])
        return F32(s / F32(len(idx)))
    rxs, rys, lxs, lys = mean(geo.right, 0), mean(geo.right, L), mean(geo.left, 0), mean(geo.left, L)
    ied = F32(np.sqrt(F32(F32((rxs - lxs) * (rxs - lxs)) + F32((rys - lys) * (rys - lys)))))
    grow = F32(0)
    for lvl, rel in enumerate(geo.rel):
        g = F32(F32(F32(F32(0.5) * rel) * ied) * F32(1.1))
        if lvl > 0:
            g = F32(g + F32(F32(drift) * ied))
        grow = max(grow, g)
    grow = F32(grow + F32(4))
    xa, xb = int(np.floor(F32(minx - grow))), int(np.ceil(F32(maxx + grow)))
    ya, yb = int(np.floor(F32(miny - grow))), int(np.ceil(F32(maxy + grow)))
    xa, ya, xb, yb = max(xa, 0), max(ya, 0), min(xb, width), min(yb, height)
    if xb <= xa or yb <= ya:                                    # face entirely outside the frame
        xa, ya, xb, yb = 0, 0, min(16, width), 1
    rx = xa & ~15
    w = min(_round16(xb - rx), (row_pixels - rx) & ~15)
    return rx, ya, w, yb - ya


def frame_roi(geo, x0, frame):
    h, w, ch = frame.shape[0], frame.shape[1], _channels(frame)
    return face_roi(geo, x0, w, h, frame.strides[0] // ch)


def roi_chunks(rois):
    """detect_faces_roi's chunks: lists of face indices in caller order; None when an ROI exceeds one staging buffer."""
    chunks, used = [], 0
    for i, (_, _, w, h) in enumerate(rois):
        b = w * h
        if b > ROI_CHUNK:
            return None
        if not chunks or used + b > ROI_CHUNK:
            chunks.append([])
            used = 0
        chunks[-1].append(i)
        used += b
    return chunks


def gathers(chunks, channels):
    """roi_gather_kernel launches: per chunk, one for its grey faces and one for its colour faces."""
    return sum(len({channels[i] for i in c}) for c in chunks)


def translation_trajectory(oracle, geo, x0, s, axis=0):
    """The landmarks at which each level of a translation model computes its HOG, and the result.  Level 0's update is 0,
    every later level's is -s in x (axis 0) or y (axis 1), so x_next = x - (-s) * (1 / (1 / IED)) (sd_cascade_update's
    epilogue, float32)."""
    x = np.asarray(x0, dtype=F32).copy()
    L = x.size // 2
    levels = []
    for lvl in range(len(geo.rel)):
        levels.append(x.copy())
        if lvl > 0:
            ied = oracle.get_ied(x, geo.right, geo.left)
            inv = F32(F32(1) / F32(1.0 / ied))
            x[axis * L:(axis + 1) * L] = (x[axis * L:(axis + 1) * L] - F32(F32(-s) * inv)).astype(F32)
    return levels, x


def window_reach(oracle, geo, levels, roi, width, height):
    """How far the patch windows of these levels reach past the ROI inside the frame: the largest number of frame pixels
    by which a window crosses an ROI edge (negative: the least clearance to an ROI edge that is not a frame edge)."""
    rx, ry, rw, rh = roi
    reach = -1 << 30
    for lvl, x in enumerate(levels):
        cx, cy, half = oracle.patch_geometry(x, geo.om.hog_params[lvl], geo.right, geo.left)
        for l in range(cx.size):
            x0, y0, x1, y1 = cx[l] - half[l], cy[l] - half[l], cx[l] + half[l], cy[l] + half[l]
            fx0, fy0, fx1, fy1 = max(x0, 0), max(y0, 0), min(x1, width), min(y1, height)
            if fx0 >= fx1 or fy0 >= fy1:
                continue
            sides = []
            if rx > 0:
                sides.append(rx - fx0)
            if ry > 0:
                sides.append(ry - fy0)
            if rx + rw < width:
                sides.append(fx1 - (rx + rw))
            if ry + rh < height:
                sides.append(fy1 - (ry + rh))
            if sides:
                reach = max(reach, max(sides))
    return reach


MISS_MARGIN = 16                 # a window that crosses by this much reads a crossing pixel on every route (taps <= 5 px apart)
CLEAR_MARGIN = 3


# ---- fixtures ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def om(oracle, golden):
    return oracle.Model(golden.model_path)


@pytest.fixture(scope="module")
def geo(om):
    return Geometry(om)


@pytest.fixture(scope="module")
def model(sd, golden):
    return sd.load_detection_model(golden.model_path)


@pytest.fixture(scope="module")
def launches_per_chunk(sd, model):
    """The launches of one whole-frame chunk: a single pageable grey frame."""
    ctx = model.ctx
    frame = _grey(240, 320, 5)
    l0 = ctx.launches()
    model.detect_faces([frame], [0], boxes=[[80, 40, 150, 150]])
    return ctx.launches() - l0


def whole_frame_scene():
    """Case 1: 48 pageable frames, 1920 x 1080 colour, 1920 x 1080 grey and 1280 x 720 colour; frames 0..19 are colour
    1920 x 1080, so the first chunk (16 referenced frames) is a strided batch and the second mixes sizes.  0 to 5 faces per
    frame, some frames without faces between frames with faces, faces in shuffled order."""
    rng = np.random.default_rng(11)
    frames, face_frame, boxes = [], [], []
    for f in range(48):
        kind = 2 if f < 20 else f % 3
        h, w = (720, 1280) if kind == 1 else (1080, 1920)
        frames.append(_grey(h, w, 1000 + f) if kind == 0 else _bgr(h, w, 1000 + f))
        n = 0 if f in (3, 11, 21, 30, 31, 40) else int(rng.integers(1, 6))
        box_size = rng.integers(h // 3, h // 2 + 1, n)
        for s in box_size:
            s = int(s)
            face_frame.append(f)
            boxes.append((int(rng.integers(-s // 4, w - 3 * s // 4)), int(rng.integers(-s // 4, h - 3 * s // 4)), s, s))
    perm = rng.permutation(len(face_frame))
    return frames, np.array(face_frame, dtype=np.int32)[perm], np.array(boxes, dtype=np.int32)[perm]


def large_frames():
    """Cases 2 and 3: five 4096 x 2160 grey and five 3840 x 2160 colour frames (pageable)."""
    return [_grey(2160, 4096, 2000 + f) if f % 2 == 0 else _bgr(2160, 3840, 2000 + f) for f in range(10)]


def roi_scene(frames):
    """Case 2: 12 overlapping faces per frame with 950 .. 1250 px boxes (ROIs of 1 to 2 MB), in shuffled order."""
    rng = np.random.default_rng(12)
    face_frame, boxes = [], []
    for f, fr in enumerate(frames):
        h, w = fr.shape[:2]
        for _ in range(12):
            s = int(rng.integers(950, 1251))
            face_frame.append(f)
            boxes.append((int(rng.integers(0, w - s)), int(rng.integers(-s // 8, h - 6 * s // 5)), s, s))
    perm = rng.permutation(len(face_frame))
    return np.array(face_frame, dtype=np.int32)[perm], np.array(boxes, dtype=np.int32)[perm]


def fallback_scene(frames):
    """Case 3: 90 faces with 1000 px boxes (IED 377 px).  Every fourth face (i % 4 == 2) sits at its frame's right edge, so
    its ROI is clipped there; the others have room to drift right inside the frame.  The first and the last face are interior."""
    rng = np.random.default_rng(13)
    face_frame, boxes, edge = [], [], []
    for i in range(90):
        f = i % 10
        h, w = frames[f].shape[:2]
        at_edge = i % 4 == 2
        x = w - 900 if at_edge else int(rng.integers(100, w - 2400))
        face_frame.append(f)
        boxes.append((x, int(rng.integers(0, h - 1100)), 1000, 1000))
        edge.append(at_edge)
    return np.array(face_frame, dtype=np.int32), np.array(boxes, dtype=np.int32), np.array(edge)


def upload_scene():
    """Case 7: 20 colour frames of 480 x 640..643, one of 4000 x 4096 (its B,G,R alone closes the first 64 MiB chunk), then
    nine of 1080 x 1918..1920: 123 MB of B,G,R in three chunks, the second larger than the first."""
    frames = [_bgr(480, 640 + i % 4, 3000 + i) for i in range(20)]
    frames.append(_bgr(4000, 4096, 3020))
    frames += [_bgr(1080, 1920 - i % 3, 3021 + i) for i in range(9)]
    return frames


def upload_chunks(frames):
    """sd_upload_frames's chunks: (first, end, B,G,R bytes)."""
    out, i0 = [], 0
    while i0 < len(frames):
        b, i1 = full_bytes(frames[i0]) - frames[i0].shape[0] * _round16(frames[i0].shape[1]), i0 + 1
        while i1 < len(frames):
            nb = frames[i1].shape[0] * _round16(3 * frames[i1].shape[1])
            if b + nb > UPLOAD_CHUNK:
                break
            b += nb
            i1 += 1
        out.append((i0, i1, b))
        i0 = i1
    return out


def _x0(sd, model, boxes):
    return np.stack([sd.align_mean(model.get_mean(), b) for b in boxes]).astype(F32)


def _align_mean(oracle, om, boxes):
    return np.stack([oracle.align_mean(om.mean, b) for b in boxes]).astype(F32)


# ---- host-only checks of the scenes ------------------------------------------------------------------------------------
def test_whole_frame_scene_spans_three_chunks_of_both_kinds():
    frames, face_frame, _ = whole_frame_scene()
    chunks = full_chunks(frames, face_frame)
    assert len(chunks) >= 3
    shapes = [{frames[f].shape[:2] for f in c} for c in chunks]
    assert len(shapes[0]) == 1 and any(len(s) > 1 for s in shapes[1:])           # strided batch, then descriptors
    counts = np.bincount(face_frame, minlength=len(frames))
    assert counts.max() == 5
    empty = np.flatnonzero(counts == 0)
    assert any(0 < f < len(frames) - 1 and counts[f - 1] and counts[f + 1] for f in empty)
    assert not np.all(np.diff(face_frame) >= 0)                                   # shuffled
    print(f"\nwhole-frame chunks {len(chunks)}: frames {[len(c) for c in chunks]}, "
          f"MB {[round(sum(full_bytes(frames[f]) for f in c) / 1e6, 1) for c in chunks]}")


def test_roi_scene_spans_three_chunks_with_both_gathers(oracle, om, geo):
    frames = large_frames()
    face_frame, boxes = roi_scene(frames)
    x0 = _align_mean(oracle, om, boxes)
    rois = [face_roi(geo, x0[i], frames[f].shape[1], frames[f].shape[0], frames[f].shape[1]) for i, f in enumerate(face_frame)]
    sizes = [w * h for _, _, w, h in rois]
    assert 1e6 <= min(sizes) and max(sizes) <= 2 * MiB
    chunks = roi_chunks(rois)
    channels = [_channels(frames[f]) for f in face_frame]
    assert len(chunks) >= 3 and gathers(chunks, channels) == 2 * len(chunks)
    print(f"\nROI chunks {len(chunks)}: faces {[len(c) for c in chunks]}")


def _fallback_plan(oracle, geo, frames, face_frame, boxes, s):
    """(faces expected to fall back, least margin of the decision in pixels)."""
    x0 = np.stack([oracle.align_mean(geo.om.mean, b) for b in boxes]).astype(F32)
    miss, margin = [], 1 << 30
    for i, f in enumerate(face_frame):
        h, w = frames[f].shape[:2]
        levels, _ = translation_trajectory(oracle, geo, x0[i], s)
        reach = window_reach(oracle, geo, levels, face_roi(geo, x0[i], w, h, w), w, h)
        if reach >= MISS_MARGIN:
            miss.append(i)
            margin = min(margin, reach)
        else:
            assert reach <= -CLEAR_MARGIN, (i, s, reach)                          # no face near the decision
            margin = min(margin, -reach)
    return miss, margin


def test_fallback_scene_is_decided_in_closed_form(oracle, om, geo):
    frames = large_frames()
    face_frame, boxes, edge = fallback_scene(frames)
    x0 = _align_mean(oracle, om, boxes)
    assert min(oracle.get_ied(x, geo.right, geo.left) for x in x0) >= 150
    miss, margin = _fallback_plan(oracle, geo, frames, face_frame, boxes, 0.6)
    assert miss == [i for i in range(len(edge)) if not edge[i]]                   # interior faces miss, edge faces do not
    assert _fallback_plan(oracle, geo, frames, face_frame, boxes, 0.1)[0] == []
    rois = [face_roi(geo, x0[i], frames[f].shape[1], frames[f].shape[0], frames[f].shape[1]) for i, f in enumerate(face_frame)]
    assert all(r[0] + r[2] == frames[face_frame[i]].shape[1] for i, r in enumerate(rois) if edge[i])
    chunks = roi_chunks(rois)
    assert len(chunks) >= 2 and all(any(i in miss for i in c) for c in chunks)
    assert miss[0] == 0 and miss[-1] == len(face_frame) - 1
    print(f"\nfallback scene: {len(miss)} expected fallbacks over {len(chunks)} ROI chunks, least margin {margin} px")


def test_upload_scene_grows_its_scratch_across_three_chunks():
    frames = upload_scene()
    chunks = upload_chunks(frames)
    assert len(chunks) >= 3 and sum(b for _, _, b in chunks) > UPLOAD_CHUNK
    assert chunks[1][2] > chunks[0][2] * 9 // 8                                   # past the workspace's 1/8 slack: it grows
    assert {f.shape[1] % 4 for f in frames} == {0, 1, 2, 3}
    print(f"\nupload chunks: {[(a, b, round(c / 1e6, 1)) for a, b, c in chunks]}")


# ---- GPU: case 1, the whole-frame route over three chunks --------------------------------------------------------------
def _resident_reference(sd, model, frames, face_frame, x0, faces):
    """detect_batch_device over the referenced frames, converted once and resident whole, per frame size, with an image
    index: (F, 2L) for `faces`."""
    out = np.empty((len(faces), x0.shape[1]), dtype=F32)
    sizes = sorted({frames[face_frame[i]].shape[:2] for i in faces})
    for size in sizes:
        sel = [k for k, i in enumerate(faces) if frames[face_frame[i]].shape[:2] == size]
        fids = sorted({int(face_frame[faces[k]]) for k in sel})
        dev = torch.stack([sd.bgr2gray(frames[f])[0] if frames[f].ndim == 3 else torch.from_numpy(frames[f]).cuda()
                           for f in fids])
        index = np.array([fids.index(face_frame[faces[k]]) for k in sel], dtype=np.int32)
        got = model.detect_batch_device(dev, torch.from_numpy(x0[[faces[k] for k in sel]]).cuda(), image_index=index)
        out[sel] = got.cpu().numpy()
        del dev
    return out


def _check_oracle(oracle, om, frames, face_frame, boxes, x0, got, faces):
    for i in faces:
        f = frames[face_frame[i]]
        gray = oracle.bgr2gray_u8(f) if f.ndim == 3 else f
        ref = om.detect_batch(gray[None], boxes[i:i + 1])[0]
        err = np.max(np.abs(got[i] - ref)) / np.max(np.abs(ref))
        if err > 1e-4:                                            # a face on a rounding tie (see test_gpu_detect)
            near = _rounding_margin(oracle, om, gray, x0[i])
            print(f"face {i}: rel err {err:.2e}, rounding margin {near:.2e}")
            assert near <= 5e-5 and np.max(np.abs(got[i] - ref)) <= 1.0, i


@pytest.mark.gpu
def test_whole_frame_route_over_three_chunks(sd, oracle, om, model, launches_per_chunk):
    frames, face_frame, boxes = whole_frame_scene()
    chunks = full_chunks(frames, face_frame)
    colour = sum(1 for c in chunks for f in c if frames[f].ndim == 3)
    ctx = model.ctx
    l0, fb0 = ctx.launches(), ctx.roi_fallbacks()
    got = model.detect_faces(frames, face_frame, boxes=boxes)
    launches = ctx.launches() - l0
    print(f"\nwhole-frame route: {len(face_frame)} faces, {len(chunks)} chunks, {launches} launches "
          f"({launches_per_chunk} per chunk + {colour} colour conversions)")
    assert len(chunks) >= 3
    assert launches == len(chunks) * launches_per_chunk + colour
    assert ctx.roi_fallbacks() == fb0
    x0 = _x0(sd, model, boxes)
    ref = _resident_reference(sd, model, frames, face_frame, x0, list(range(len(face_frame))))
    bad = np.flatnonzero(np.any(got.view(np.uint32) != ref.view(np.uint32), axis=1))
    assert bad.size == 0, f"faces {bad.tolist()[:10]} (frames {face_frame[bad].tolist()[:10]}) differ from the resident reference"
    # the oracle on a face of each chunk, from its first and its last frame
    pick = []
    for c in chunks:
        for f in (c[0], c[-1]):
            pick.append(int(np.flatnonzero(face_frame == f)[0]))
    _check_oracle(oracle, om, frames, face_frame, boxes, x0, got, sorted(set(pick)))


# ---- GPU: cases 2 and 3, the ROI route over three chunks and its fallbacks ---------------------------------------------
@pytest.fixture(scope="module")
def large(sd):
    frames = large_frames()
    pin = Pinned(sd)
    pinned = [pin(f) for f in frames]
    yield frames, pinned
    del pinned
    pin.release()


@pytest.mark.gpu
def test_roi_route_over_three_chunks(sd, oracle, om, geo, model, large, launches_per_chunk):
    frames, pinned = large
    face_frame, boxes = roi_scene(frames)
    x0 = _x0(sd, model, boxes)
    rois = [frame_roi(geo, x0[i], pinned[f]) for i, f in enumerate(face_frame)]
    chunks = roi_chunks(rois)
    n_gathers = gathers(chunks, [_channels(frames[f]) for f in face_frame])
    ctx = model.ctx
    l0, fb0 = ctx.launches(), ctx.roi_fallbacks()
    got = model.detect_faces(pinned, face_frame, boxes=boxes)
    launches, fb = ctx.launches() - l0, ctx.roi_fallbacks() - fb0
    print(f"\nROI route: {len(face_frame)} faces, {len(chunks)} chunks, {n_gathers} gathers, {launches} launches, "
          f"ROI fallbacks {fb}, pinned {Pinned.held / 1e6:.0f} MB")
    assert len(chunks) >= 3
    assert fb == 0, "a face of this scene left its ROI: the launch count below assumes none does"
    assert launches == len(chunks) * launches_per_chunk + n_gathers
    full = model.detect_faces(frames, face_frame, boxes=boxes)
    assert np.array_equal(got.view(np.uint32), full.view(np.uint32))
    ref = _resident_reference(sd, model, frames, face_frame, x0, list(range(len(face_frame))))
    bad = np.flatnonzero(np.any(got.view(np.uint32) != ref.view(np.uint32), axis=1))
    assert bad.size == 0, f"faces {bad.tolist()[:10]} differ from the resident reference"
    # the oracle on the first and the last face of each chunk
    _check_oracle(oracle, om, frames, face_frame, boxes, x0, got, sorted({i for c in chunks for i in (c[0], c[-1])}))


def _translation_model(sd, model, om, s, axis=0):
    """The golden model's mean, ids and HOG parameters; every regressor weight 0 except the bias row's x (axis 0) or y entries,
    0 at level 0 and -s after it, so that each level after the first moves every landmark s inter-eye distances to the right
    (or down)."""
    regs = []
    for lvl in range(model.num_levels):
        D, P = model.weights(lvl).shape
        w = np.zeros((D, P), dtype=F32)
        if lvl > 0:
            w[-1, axis * (P // 2):(axis + 1) * (P // 2)] = -s
        r = sd.LinearRegressor(ctx=model.ctx)
        r.x = torch.from_numpy(w).cuda()
        regs.append(r)
    opt = sd.SupervisedDescentOptimiser(regs, ctx=model.ctx)
    return sd.detection_model.from_parts(opt, model.get_mean(), model.landmark_ids,
                                         [model.hog_param(lvl) for lvl in range(model.num_levels)], om.right_ids, om.left_ids,
                                         ctx=model.ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("s", [0.6, 0.1])
def test_roi_fallbacks_across_chunks(sd, oracle, om, geo, model, large, s):
    """Interior faces drift 0.6 IED per level, past face_roi's allowance of 0.2 IED, and must fall back; faces whose ROI is
    clipped at the frame's right edge drift out of the frame, not out of the ROI, and must not; at 0.1 IED per level none
    may.  The fallback faces lie in every ROI chunk and at both ends of the caller's order."""
    frames, pinned = large
    face_frame, boxes, edge = fallback_scene(frames)
    miss, margin = _fallback_plan(oracle, geo, frames, face_frame, boxes, s)
    tm = _translation_model(sd, model, om, s)
    ctx = model.ctx
    fb0 = ctx.roi_fallbacks()
    got = tm.detect_faces(pinned, face_frame, boxes=boxes)
    fb = ctx.roi_fallbacks() - fb0
    x0 = _x0(sd, model, boxes)
    rois = [frame_roi(geo, x0[i], pinned[f]) for i, f in enumerate(face_frame)]
    print(f"\ns = {s}: ROI fallbacks {fb}, expected {len(miss)} (least margin {margin} px), ROI chunks {len(roi_chunks(rois))}")
    assert fb == len(miss)
    full = tm.detect_faces(frames, face_frame, boxes=boxes)
    assert ctx.roi_fallbacks() - fb0 == fb
    assert np.array_equal(got.view(np.uint32), full.view(np.uint32))
    # the closed form: x moved by 3 s IED, y unchanged
    for i in range(len(face_frame)):
        _, want = translation_trajectory(oracle, geo, x0[i], s)
        assert np.max(np.abs(got[i] - want)) <= 1e-3, i
    del tm


@pytest.mark.gpu
def test_drift_allowance_of_face_roi(sd, oracle, om, geo, model):
    """face_roi grows the ROI by the largest of the levels' half patch (x 1.1) plus 0.2 IED after level 0: 0.585 IED for the
    golden model, against 0.55 IED without the allowance.  A face with an IED of 2400 px moved down 0.22125 IED per level
    reaches 0.5675 IED at level 3: inside the ROI with the allowance, tens of pixels past it without."""
    frame = _grey(8192, 8192, 4001)
    boxes = np.array([[500, -2200, 6400, 6400]], dtype=np.int32)
    s = 0.22125
    x0 = _x0(sd, model, boxes)
    assert oracle.get_ied(x0[0], geo.right, geo.left) >= 2400
    levels, want = translation_trajectory(oracle, geo, x0[0], s, axis=1)
    roi = face_roi(geo, x0[0], 8192, 8192, 8192)
    bare = face_roi(geo, x0[0], 8192, 8192, 8192, drift=0.0)
    assert roi[2] * roi[3] < ROI_CHUNK
    P3 = 2 * oracle.patch_geometry(levels[-1], om.hog_params[-1], geo.right, geo.left)[2].max()
    fs3 = om.hog_params[-1].num_cells * om.hog_params[-1].cell_size
    inside, outside = window_reach(oracle, geo, levels, roi, 8192, 8192), window_reach(oracle, geo, levels, bare, 8192, 8192)
    print(f"\ndrift allowance: level-3 windows {-inside} px inside the ROI, {outside} px past it without the allowance")
    assert inside <= -CLEAR_MARGIN and outside >= MISS_MARGIN + -(-P3 // fs3)      # taps of the last level lie P / fs apart
    pin = Pinned(sd)
    pinned = pin(frame)
    tm = _translation_model(sd, model, om, s, axis=1)
    ctx = model.ctx
    fb0 = ctx.roi_fallbacks()
    got = tm.detect_faces([pinned], [0], boxes=boxes)
    assert ctx.roi_fallbacks() == fb0
    assert np.array_equal(got.view(np.uint32), tm.detect_faces([frame], [0], boxes=boxes).view(np.uint32))
    assert np.max(np.abs(got[0] - want)) <= 1e-3
    del tm, pinned
    pin.release()


# ---- GPU: case 4, an ROI larger than a staging buffer ------------------------------------------------------------------
@pytest.mark.gpu
def test_roi_larger_than_a_staging_buffer_takes_the_whole_frame_route(sd, geo, model, launches_per_chunk):
    frame = _grey(8192, 8192, 4000)
    boxes = np.array([[300, 300, 600, 600], [400, -700, 7000, 7000], [7000, 7200, 700, 700]], dtype=np.int32)
    pin = Pinned(sd)
    pinned = pin(frame)
    x0 = _x0(sd, model, boxes)
    rois = [frame_roi(geo, x, pinned) for x in x0]
    assert rois[1][2] * rois[1][3] > ROI_CHUNK + MiB and max(r[2] * r[3] for r in (rois[0], rois[2])) < ROI_CHUNK
    assert roi_chunks(rois) is None
    ctx = model.ctx
    l0, fb0 = ctx.launches(), ctx.roi_fallbacks()
    got = model.detect_faces([pinned], [0, 0, 0], boxes=boxes)
    launches, fb = ctx.launches() - l0, ctx.roi_fallbacks() - fb0
    print(f"\nROI of {rois[1][2] * rois[1][3] / MiB:.1f} MiB: {launches} launches, ROI fallbacks {fb}, "
          f"pinned {Pinned.held / 1e6:.0f} MB (peak {Pinned.peak / 1e6:.0f} MB)")
    assert launches == launches_per_chunk and fb == 0                             # one whole-frame chunk, no gather
    full = model.detect_faces([frame], [0, 0, 0], boxes=boxes)
    assert np.array_equal(got.view(np.uint32), full.view(np.uint32))
    del pinned
    pin.release()


# ---- GPU: case 5, the ROI route's edges ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_roi_edges_match_the_whole_frame_route(sd, oracle, om, geo, model):
    pin = Pinned(sd)
    ctx = model.ctx

    def both(frames, face_frame, boxes, pitches):
        pinned = [pin(f, p) for f, p in zip(frames, pitches)]
        fb0 = ctx.roi_fallbacks()
        got = model.detect_faces(pinned, face_frame, boxes=boxes)
        fb = ctx.roi_fallbacks() - fb0
        full = model.detect_faces(frames, face_frame, boxes=boxes)
        assert np.array_equal(got.view(np.uint32), full.view(np.uint32))
        return pinned, fb

    # a colour frame of width 200 at pitch round16(600) = 608: an ROI ends by x = 192 (608 / 3 = 202 pixels a row, in whole
    # 16-pixel steps), so a face whose level-0 windows reach past x = 192 must fall back
    colour = _bgr(240, 200, 5000)
    boxes = np.array([[60, 20, 180, 180], [-20, 30, 150, 150], [90, 60, 120, 120]], dtype=np.int32)
    x0 = _x0(sd, model, boxes)
    pinned, fb = both([colour], [0, 0, 0], boxes, [608])
    rois = [frame_roi(geo, x, pinned[0]) for x in x0]
    assert max(r[0] + r[2] for r in rois) == 192
    # level 0 resizes these windows by less than 2 (P <= 2 fs, fs = 55), so its taps read every column but perhaps the last: a
    # level-0 window that reaches
    # 4 pixels past x = 192 reads a pixel outside its ROI
    assert all(2 * oracle.patch_geometry(x, om.hog_params[0], geo.right, geo.left)[2].max() <= 2 * 55 for x in x0)
    must = [i for i in range(3) if window_reach(oracle, geo, [x0[i]], rois[i], 200, 240) >= 4]
    print(f"\nright border of a colour row: ROIs {rois}, ROI fallbacks {fb} (at least {len(must)})")
    assert must and fb >= len(must)
    # frames narrower than 16 pixels: grey at a 16-byte pitch (an ROI of 16 pixels), colour at 32 (no whole 16-pixel step)
    narrow = [_grey(240, 12, 5001), _bgr(240, 10, 5002)]
    boxes = np.array([[-80, 20, 160, 160], [-70, 40, 150, 150], [-90, 10, 170, 170]], dtype=np.int32)
    pinned, fb = both(narrow, [0, 1, 1], boxes, [16, 32])
    rois = [frame_roi(geo, x, pinned[f]) for x, f in zip(_x0(sd, model, boxes), [0, 1, 1])]
    print(f"frames narrower than 16 px: ROIs {rois}, ROI fallbacks {fb}")
    assert rois[0][2] == 16 and rois[1][2] == 0 and fb >= 2
    # a face entirely outside its frame (face_roi's empty branch) beside one inside it
    grey = _grey(240, 320, 5003)
    boxes = np.array([[1000, 900, 150, 150], [80, 40, 150, 150], [-600, -500, 200, 200]], dtype=np.int32)
    pinned, fb = both([grey], [0, 0, 0], boxes, [320])
    rois = [frame_roi(geo, x, pinned[0]) for x in _x0(sd, model, boxes)]
    print(f"faces outside the frame: ROIs {rois}, ROI fallbacks {fb}")
    assert rois[0] == (0, 0, 16, 1) and rois[2] == (0, 0, 16, 1)
    pin.release()


# ---- GPU: case 6, the miss flag at the ROI's exact edge ------------------------------------------------------------------
CFG = (1, 5, 6, 4)               # fs = 30
ROI = (48, 50, 315, 221)         # inside the 400 x 320 frame on every side; 315 wide, so a 320 or 324 byte pitch has guard bytes
P_STAGED, P_UNSTAGED = 40, 150   # 150 = 5 fs: every x tap pair has a right tap of weight 0


def resize_taps(fs, P):
    """hog_resize_tap restated: per output index, (source index, weight of the right / lower tap), and the lower index."""
    inv = fs / P
    scale = 1.0 / inv
    out = []
    for t in range(fs):
        f = F32((t + 0.5) * scale - 0.5)
        s = int(np.floor(f))
        f = F32(f - F32(s))
        sx, fx = s, f
        if sx < 0:
            sx, fx = 0, F32(0)
        if sx >= P - 1:
            sx, fx = P - 1, F32(0)
        w1 = int(np.rint(F32(fx * F32(2048))))
        out.append((sx, w1, min(max(s, 0), P - 1), min(max(s + 1, 0), P - 1)))
    return out


def read_pixels(P, fs, staged):
    """(columns, rows) of a P x P window that the kernel reads: every pixel through the staged load loops; through the unstaged
    route, the taps -- a right tap of weight 0 is skipped, a lower tap of weight 0 is read."""
    if staged:
        return set(range(P)), set(range(P))
    taps = resize_taps(fs, P)
    cols = {sx for sx, _, _, _ in taps} | {sx + 1 for sx, w1, _, _ in taps if w1 != 0}
    rows = {y for _, _, y0, y1 in taps for y in (y0, y1)}
    return cols, rows


def flag_expected(P, fs, staged, x0, y0, roi, width, height):
    rx, ry, rw, rh = roi
    cols, rows = read_pixels(P, fs, staged)
    xs = [x0 + c for c in cols if 0 <= x0 + c < width]
    ys = [y0 + r for r in rows if 0 <= y0 + r < height]
    return bool(xs and ys and (min(xs) < rx or max(xs) >= rx + rw or min(ys) < ry or max(ys) >= ry + rh))


def edge_windows(P, fs, staged):
    """(name, x0, y0) of windows that end exactly on each ROI edge, cross each edge by one pixel and, through the unstaged
    route, put their outermost read tap just inside or just outside each edge."""
    rx, ry, rw, rh = ROI
    mx, my = rx + (rw - P) // 2, ry + (rh - P) // 2
    wins = [("on left", rx, my), ("on right", rx + rw - P, my), ("on top", mx, ry), ("on bottom", mx, ry + rh - P),
            ("over left", rx - 1, my), ("over right", rx + rw - P + 1, my), ("over top", mx, ry - 1),
            ("over bottom", mx, ry + rh - P + 1)]
    if not staged:
        cols, rows = read_pixels(P, fs, False)
        c0, c1, r0, r1 = min(cols), max(cols), min(rows), max(rows)
        wins += [("tap on left", rx - c0, my), ("tap over left", rx - 1 - c0, my),
                 ("tap on right", rx + rw - 1 - c1, my), ("tap over right", rx + rw - c1, my),
                 ("zero-weight right tap over right", rx + rw - (c1 + 1), my),
                 ("tap on top", mx, ry - r0), ("tap over top", mx, ry - 1 - r0),
                 ("tap on bottom", mx, ry + rh - 1 - r1), ("tap over bottom", mx, ry + rh - r1)]
    return wins


def _words_layout(lay):
    """The same ROIs at a pitch of 4 mod 16: resident windows take the word loop instead of the 16-byte one."""
    o = 0
    for i in range(len(lay.frames)):
        lay.pitches[i] = _round16(lay.rois[i][2]) + 4
        lay.offsets[i] = o
        o = _round16(o + lay.pitches[i] * lay.rois[i][3])
        lay.desc[i]["align"] = lay.offsets[i] | lay.pitches[i]
    lay.total = o
    return lay


@pytest.mark.gpu
def test_roi_miss_flag_at_the_exact_roi_edge(sd, oracle):
    """One ROI per sample, so that each flag belongs to one window.  Staged windows that end on an ROI edge are resident
    (16-byte or word loads by the layout's alignment) and do not flag; windows that cross an edge by one pixel take the
    byte loop and flag.  The unstaged route reads only the resize taps: a right tap of weight 0 is never read and cannot
    flag, the lower tap of a row pair is read even at weight 0 and flags; the rule is checked window by window."""
    fs = CFG[1] * CFG[2]
    cap = smem_layout(CFG)[0]
    assert ((P_STAGED + 30) & ~15) * P_STAGED <= cap < ((P_UNSTAGED + 30) & ~15) * P_UNSTAGED
    assert P_STAGED <= largest_staged(cap) < P_UNSTAGED
    frame = _frames()[0]
    rx, ry, rw, rh = ROI
    assert rx > 0 and ry > 0 and rx + rw + 1 < KW and ry + rh + 1 < KH
    ctx = sd.default_context()
    samples, names, expected = [], [], []
    for P, staged, eyes in ((P_STAGED, True, (150, 160)), (P_UNSTAGED, False, (130, 160))):
        for name, x0, y0 in edge_windows(P, fs, staged):
            samples.append(_sample(len(samples), P, (x0, y0), (x0, y0), eyes=eyes))
            names.append(f"P={P} {name}")
            expected.append(flag_expected(P, fs, staged, x0, y0, ROI, KW, KH))
        ex, ey = eyes                                             # the eyes' windows are resident
        assert not flag_expected(P, fs, staged, ex - P // 2, ey - P // 2, (rx, ry, rw - P, rh), KW, KH)
    taps = resize_taps(fs, P_UNSTAGED)
    assert any(w1 == 0 for _, w1, _, _ in taps)
    exp = dict(zip(names, expected))
    for side in ("left", "right", "top", "bottom"):
        assert exp[f"P={P_STAGED} over {side}"] and not exp[f"P={P_STAGED} on {side}"]
        assert exp[f"P={P_UNSTAGED} tap over {side}"] and not exp[f"P={P_UNSTAGED} tap on {side}"]
    assert not exp[f"P={P_UNSTAGED} zero-weight right tap over right"]
    # the last row read is the lower tap of the last output row, at weight 0 ("tap over bottom" puts it past the ROI)
    sx, w1, y0, y1 = taps[-1]
    assert w1 == 0 and y1 == max(read_pixels(P_UNSTAGED, fs, False)[1]) and exp[f"P={P_UNSTAGED} tap over bottom"]
    frames = [frame] * len(samples)
    want = truth(oracle, frames, samples, CFG)
    bad = []
    for kind in ("vec16", "words"):
        lay = Layout("roi", frames, [ROI] * len(samples))
        if kind == "words":
            lay = _words_layout(lay)
        assert all((d["align"] % 16 == 0) == (kind == "vec16") and d["align"] % 4 == 0 for d in lay.desc)
        ib, keep, miss = device_batch(lay)
        got = run_kernel(ctx, ib, samples, CFG)
        flags = miss.cpu().numpy().astype(bool).tolist()
        for n, e, g in zip(names, expected, flags):
            if e != g:
                bad.append(f"{kind}: {n}: flag {g}, expected {e}")
        keep_rows = [i for i, e in enumerate(expected) if not e]
        b, worst = compare(tuple(a[keep_rows] for a in got), tuple(a[keep_rows] for a in want), f"{kind} unflagged windows")
        bad += b
        print(f"\n{kind}: {sum(flags)} of {len(flags)} windows flagged, unflagged windows' worst feature error {worst:.2e} "
              f"(tolerance {FEATURE_TOL:g})")
        del keep
    assert not bad, "\n".join(bad)


# ---- GPU: case 7, sd_upload_frames over three colour chunks ------------------------------------------------------------
@pytest.mark.gpu
def test_upload_frames_over_three_colour_chunks(sd, oracle, om, model):
    """A fresh context, so that its B,G,R scratch starts empty and grows at the second chunk."""
    frames = upload_scene()
    chunks = upload_chunks(frames)
    ctx = sd.Context(0)
    recs, keep = sd._host_frames(frames)
    l0 = ctx.launches()
    buf, ib = sd._upload_host_frames(recs, ctx)
    assert ctx.launches() - l0 == len(frames)                   # one colour conversion per frame
    host = buf.cpu().numpy()
    off = 0
    for i, f in enumerate(frames):
        h, w = f.shape[:2]
        got = host[off:off + h * _round16(w)].reshape(h, _round16(w))[:, :w]
        assert np.array_equal(got, oracle.bgr2gray_u8(f)), i
        off += h * _round16(w)
    print(f"\nupload: {len(frames)} colour frames in {len(chunks)} chunks of {[round(b / 1e6, 1) for _, _, b in chunks]} MB")
    del buf
    # HogTransform over all frames at once against one over each frame alone
    hp = [model.hog_param(lvl) for lvl in range(model.num_levels)]
    rng = np.random.default_rng(7)
    boxes = []
    for f in frames:
        h, w = f.shape[:2]
        s = int(rng.integers(min(h, w) // 3, min(h, w) // 2 + 1))
        boxes.append((int(rng.integers(-s // 4, w - 3 * s // 4)), int(rng.integers(-s // 4, h - 3 * s // 4)), s, s))
    x = _x0(sd, model, boxes)
    together = sd.HogTransform(frames, hp, om.landmark_ids, om.right_ids, om.left_ids, ctx=ctx)
    for lvl in (0, model.num_levels - 1):
        rows = together(x, lvl, np.arange(len(frames))).cpu().numpy()
        for i, f in enumerate(frames):
            alone = sd.HogTransform([f], hp, om.landmark_ids, om.right_ids, om.left_ids, ctx=ctx)
            one = alone(x[i:i + 1], lvl, [0]).cpu().numpy()
            assert np.array_equal(rows[i].view(np.uint32), one[0].view(np.uint32)), (lvl, i)
    del together
    ctx.close()
