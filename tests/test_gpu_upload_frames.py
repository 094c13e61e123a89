"""sd_upload_frames: host frames of any sizes and row steps, grey or colour, into the grey batch sd_hog_batch reads."""
import ctypes as C

import numpy as np
import pytest
import torch

import synth
from test_gpu_detect_frames import _colour, _pinned

pytestmark = pytest.mark.gpu

FRAME = np.dtype([("w", "<i4"), ("h", "<i4"), ("s", "<i4"), ("r", "<i4"), ("o", "<i8")])


def _round16(v):
    return (v + 15) // 16 * 16


def _padded(frame, pad):
    """A pageable view of `frame` whose rows are `pad` pixels longer than the frame."""
    h, w = frame.shape[:2]
    buf = np.zeros((h, w + pad) + frame.shape[2:], dtype=np.uint8)
    buf[:, :w] = frame
    return buf[:, :w]


def _rec(sd, a):
    a = a.numpy() if isinstance(a, torch.Tensor) else a
    return sd.HostFrameC(a.ctypes.data, a.shape[1], a.shape[0], a.strides[0], 1 if a.ndim == 2 else a.shape[2])


def _upload(sd, recs, buf=None, nbytes=None):
    """(status, bytes, ImageBatchC); buf None = the size query."""
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    table = (sd.HostFrameC * max(len(recs), 1))(*recs)
    size = C.c_size_t(0 if nbytes is None else nbytes)
    ib = sd.ImageBatchC()
    rc = _capi.lib().sd_upload_frames(ctx.h, table, len(recs), None if buf is None else C.c_void_p(buf), C.byref(size), C.byref(ib))
    return rc, size.value, ib


def _check_frames(buf, ib, grays, table_at):
    """Every frame's grey bytes at its descriptor's offset and pitch; the sd_frame table {w, h, round16(w), 0, offset}."""
    host = buf.cpu().numpy()
    table = host[table_at:table_at + len(grays) * FRAME.itemsize].view(FRAME)
    off = 0
    for i, g in enumerate(grays):
        h, w = g.shape
        assert tuple(table[i]) == (w, h, _round16(w), 0, off), i
        got = host[off:off + h * _round16(w)].reshape(h, _round16(w))[:, :w]
        assert np.array_equal(got, g), i
        off += h * _round16(w)
    assert table_at == off and ib.d_frames == buf.data_ptr() + off and ib.d_data == buf.data_ptr() and ib.count == len(grays)


def test_frames_of_three_sizes_grey_and_colour(sd, oracle):
    sizes = [(37, 45), (50, 70), (29, 101)]                   # no width a multiple of 16
    frames = []
    for i in range(6):
        h, w = sizes[i % 3]
        frames.append(_colour(h, w, seed=60 + 5 * i) if i % 2 else synth.smooth_images(1, h, w, seed=60 + 5 * i)[0])
    grays = [oracle.bgr2gray_u8(f) if f.ndim == 3 else f for f in frames]
    for name, host in (("pageable", [_padded(f, 3 * i) for i, f in enumerate(frames)]), ("pinned", [_pinned(f) for f in frames])):
        recs = [_rec(sd, a) for a in host]
        rc, need, _ = _upload(sd, recs)
        assert rc == 0 and need == sum(h * _round16(w) for h, w in (g.shape for g in grays)) + FRAME.itemsize * len(frames), name
        buf = torch.empty(need, dtype=torch.uint8, device="cuda")
        rc, _, ib = _upload(sd, recs, buf.data_ptr(), need)
        assert rc == 0, name
        _check_frames(buf, ib, grays, need - FRAME.itemsize * len(frames))


def test_equal_sizes_give_a_plain_batch(sd, oracle):
    frames = [_colour(33, 50, seed=80), synth.smooth_images(1, 33, 50, seed=81)[0], _padded(_colour(33, 50, seed=82), 7)]
    grays = [oracle.bgr2gray_u8(f) if f.ndim == 3 else f for f in frames]
    recs = [_rec(sd, a) for a in frames]
    rc, need, _ = _upload(sd, recs)
    assert rc == 0 and need == 3 * 33 * 64
    buf = torch.empty(need, dtype=torch.uint8, device="cuda")
    rc, _, ib = _upload(sd, recs, buf.data_ptr(), need)
    assert rc == 0 and not ib.d_frames and ib.d_data == buf.data_ptr()
    assert (ib.width, ib.height, ib.row_stride, ib.image_stride, ib.count) == (50, 33, 64, 33 * 64, 3)
    got = buf.cpu().numpy().reshape(3, 33, 64)[:, :, :50]
    assert np.array_equal(got, np.stack(grays))


def test_invalid_inputs_leave_the_buffer(sd):
    grey = synth.smooth_images(1, 40, 52, seed=90)[0]
    colour = _colour(30, 20, seed=91)
    good = [_rec(sd, grey), _rec(sd, colour)]
    rc, need, _ = _upload(sd, good)
    assert rc == 0
    buf = torch.full((need + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    base = buf.data_ptr()
    two = sd.HostFrameC(grey.ctypes.data, 26, 40, 52, 2)
    short = sd.HostFrameC(colour.ctypes.data, 20, 30, 59, 3)
    null = sd.HostFrameC(None, 52, 40, 52, 1)
    cases = {
        "one byte short": (good, base, need - 1),
        "two channels": ([good[0], two], base, need),
        "row_stride < width * channels": ([good[0], short], base, need),
        "null pointer": ([null, good[1]], base, need),
        "unaligned d_buf": (good, base + 1, need),
        "no frames": ([], base, need),
    }
    for name, (recs, ptr, nbytes) in cases.items():
        assert _upload(sd, recs, ptr, nbytes)[0] == 1, name     # SD_ERR_INVALID
        assert torch.all(buf == 0xA5), name
    for name in ("two channels", "row_stride < width * channels", "null pointer", "no frames"):
        assert _upload(sd, cases[name][0])[0] == 1, name       # the size query checks the frames too
    assert _upload(sd, good, base, need)[0] == 0              # the context still works
