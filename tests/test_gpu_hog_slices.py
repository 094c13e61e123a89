"""The dense-HOG and sliding-window kernels where their work is cut up, against the same items computed alone.

- Launch chunks of 65,535 frames (grid z): sd_hog_dense (TMA route and frame table), sd_hog_dense_images, sd_hog_dense_polar,
  sd_hog_pyramid's dense pass, sd_hog_relayout and sd_hog_render on batches of N = 65,535 + 2 P + 3 items, item i being base
  item i mod P.  P = 7 is coprime with 65,535 = 3 * 5 * 17 * 257, so a chunk that read item blockIdx.z in place of
  frame0 + blockIdx.z would read a different base item.  Every item equals its base item computed alone, bit for bit; the
  canaries around and between the results survive; ctx.launches() shows that the call made two launches of the chunked
  kernel.  The alone results of the feature kernels are themselves within tests/hog_ref64.py's float64 bars.
- Pyramid slices of 64 MB of level pixels: several slices with a scratch that grows between them, a frame whose levels alone
  exceed a slice, and equally sized frames.  Every level equals vl_hog_pyramid of its frame alone; the frames on both sides of
  every slice boundary equal hog_dense of oracle.resize_linear_u8 of the frame; the slice count seen by ctx.launches() is the
  one the slice rule gives.
- Trainer slices of 256 MB of features: train_hog_filter over three slices, on a device batch and on a frame table, equals
  hog_train_ref.train_rule (the rule over all frames at once) bit for bit, and the two routes agree."""
import ctypes as C

import numpy as np
import pytest
import torch

import hog_ref64 as R
import hog_train_ref as T
from superviseddescent_b200 import _capi
from superviseddescent_b200._capi import FrameC, HogGridC, HogGridsC, ImageBatchC

pytestmark = pytest.mark.gpu

P = 7
N = 65535 + 2 * P + 3
CANARY = -4321.75
PYRAMID_SLICE_BYTES = 64 << 20           # level pixels per slice of sd_hog_pyramid (sd_hog_dense.cu, kPyramidSliceBytes)
TRAIN_SLICE_FLOATS = 64 << 20            # feature floats per slice of sd_hog_train_filter (sd_hog_train.cu, kSliceFloats)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _launches(sd, fn, ctx=None):
    ctx = ctx or sd.default_context()
    before = ctx.launches()
    out = fn()
    torch.cuda.synchronize()
    return out, ctx.launches() - before


def _periodic(base):
    """(N, ...) device batch whose item i is base[i mod P]"""
    idx = torch.arange(N, device="cuda") % P
    return base[idx].contiguous(), idx


def _pin(got, want, bar, what):
    r = R.worst(got, want, bar)
    assert r <= 1.0, f"{what}: error / bar {r:.3g}"
    assert np.all(got[(want == 0) & (bar == 0)] == 0), what
    return r


def _check_chunked(name, batch, alone, idx, launches):
    """batch (N, ...) against alone (P, ...) item by item, and the two launches of the chunked kernel"""
    ok = torch.equal(_bits(batch), _bits(alone)[idx])
    print(f"{name}: {N} items, {launches} launches, every item equals its base item alone: {ok}")
    assert ok, name
    assert launches == 2, (name, launches)


# ---- 65,535-item chunks ----------------------------------------------------------------------------------------------------
CS, K, VARIANT = 4, 9, 1


def test_dense_tma_route_chunks(sd):
    H = W = 16                                                    # a 16-byte row stride: the TMA route
    base = np.stack([R.blind_spot_frame(H, W, seed=40 + j, cs=CS) for j in range(P)])
    alone = torch.cat([sd.hog_dense(torch.from_numpy(base[j:j + 1]).cuda(), CS, K, VARIANT) for j in range(P)])
    worst = max(_pin(alone[j].cpu().numpy(), *R.truth(R.image_pixels(base[j], K), CS, K, VARIANT), f"base {j}") for j in range(P))
    frames, idx = _periodic(torch.from_numpy(base).cuda())
    assert frames.stride(1) == 16
    got, n = _launches(sd, lambda: sd.hog_dense(frames, CS, K, VARIANT))
    print(f"alone: worst error / bar {worst:.3f}")
    _check_chunked("sd_hog_dense tma", got, alone, idx, n)


def _scattered(out, offsets, sizes, j_of, alone):
    """Checks out at per-item offsets against alone[j] flattened, and that every float no item owns is a canary."""
    owned = torch.zeros(out.numel(), dtype=torch.bool, device="cuda")
    for j in range(P):
        items = torch.nonzero(j_of == j).flatten()
        pos = offsets[items][:, None] + torch.arange(sizes[j], device="cuda")[None]
        assert torch.equal(_bits(out[pos]), _bits(alone[j].reshape(1, -1)).expand(len(items), -1)), j
        owned[pos.flatten()] = True
    assert int(owned.sum()) == int(sum(sizes[j] for j in j_of.tolist()))
    assert bool((out[~owned] == CANARY).all())


def test_dense_frame_table_chunks(sd):
    """Two frame sizes in turn, every descriptor pointing at its base frame; results at caller offsets with 3-float gaps."""
    shapes = [(16, 16) if j % 2 == 0 else (13, 21) for j in range(P)]
    base = [R.blind_spot_frame(h, w, seed=60 + j, cs=CS) for j, (h, w) in enumerate(shapes)]
    alone = sd.hog_dense(base, CS, K, VARIANT)                    # the base frames alone, through a table of their own
    for j in range(P):
        _pin(alone[j].cpu().numpy(), *R.truth(R.image_pixels(base[j], K), CS, K, VARIANT), f"base {j}")
    data = torch.from_numpy(np.concatenate([b.ravel() for b in base])).cuda()
    starts = np.cumsum([0] + [b.size for b in base])[:-1]
    j_of = np.arange(N) % P
    table = (FrameC * N)(*[FrameC(shapes[j][1], shapes[j][0], shapes[j][1], 0, int(starts[j])) for j in j_of])
    d_table = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    sizes = [a.numel() for a in alone]
    offsets = np.cumsum([5] + [sizes[j] + 3 for j in j_of])
    out = torch.full((int(offsets[-1]) + 7,), CANARY, dtype=torch.float32, device="cuda")
    d_off = torch.from_numpy(offsets[:-1].astype(np.int64)).cuda()
    ib = ImageBatchC(C.c_void_p(data.data_ptr()), 0, 0, 0, 0, N)
    ib.d_frames = d_table.data_ptr()
    ctx = sd.default_context()
    rc, n = _launches(sd, lambda: _capi.lib().sd_hog_dense(ctx.h, C.byref(ib), CS, K, VARIANT, _capi.ptr(out), _capi.ptr(d_off)))
    assert rc == 0
    _scattered(out, d_off, sizes, torch.from_numpy(j_of).cuda(), alone)
    print(f"sd_hog_dense frame table: {N} frames, {n} launches, every frame equals its base frame alone, canaries intact")
    assert n == 2


@pytest.mark.parametrize("bil", [False, True])
def test_images_float_interleaved_chunks(sd, bil):
    H, W = 12, 13
    planar = [R.float_case_frame(3, H, W, 80 + j, CS, K, bil) for j in range(P)]
    base = np.stack([np.ascontiguousarray(np.moveaxis(f, 0, -1)) for f in planar])      # (P, H, W, 3)
    run = lambda t: sd.vl_hog(t, CS, K, VARIANT, bilinear_orientations=bil, channels_last=True)
    alone = torch.cat([run(torch.from_numpy(base[j:j + 1]).cuda()) for j in range(P)])
    for j in range(P):
        px = R.image_pixels(planar[j], K, bil, check_margin=True)
        _pin(alone[j].cpu().numpy(), *R.truth(px, CS, K, VARIANT), f"base {j}")
    frames, idx = _periodic(torch.from_numpy(base).cuda())
    got, n = _launches(sd, lambda: run(frames))
    _check_chunked(f"sd_hog_dense_images f32 x3 bilinear {bil}", got, alone, idx, n)


def test_polar_directed_bilinear_chunks(sd):
    H, W = 11, 14
    fields = [R.polar_field(H, W, seed=100 + j, K=K, directed=True, bilinear=True) for j in range(P)]
    run = lambda m, a: sd.vl_hog_polar(m, a, CS, K, VARIANT, directed=True, bilinear_orientations=True)
    alone = torch.cat([run(torch.from_numpy(m[None]).cuda(), torch.from_numpy(a[None]).cuda()) for m, a in fields])
    for j, (m, a) in enumerate(fields):
        _pin(alone[j].cpu().numpy(), *R.truth(R.polar_pixels(m, a, K, True, True), CS, K, VARIANT), f"base {j}")
    mod, idx = _periodic(torch.from_numpy(np.stack([m for m, _ in fields])).cuda())
    ang, _ = _periodic(torch.from_numpy(np.stack([a for _, a in fields])).cuda())
    got, n = _launches(sd, lambda: run(mod, ang))
    _check_chunked("sd_hog_dense_polar directed bilinear", got, alone, idx, n)


def test_pyramid_levels_past_one_chunk(sd):
    """16,400 frames of 32 x 32 at four scales: 65,600 non-empty levels in one slice, so the dense pass takes two launches."""
    scales, cs = (1.0, 0.8, 0.6, 0.5), 8
    nf = 16400
    base = np.stack([R.blind_spot_frame(32, 32, seed=120 + j, cs=cs) for j in range(P)])
    alone = []
    for j in range(P):
        feats, _ = sd.vl_hog_pyramid(torch.from_numpy(base[j:j + 1]).cuda(), scales, cs, K, VARIANT)
        assert all(v is not None for v in feats[0])
        alone.append(torch.cat([v.reshape(-1) for v in feats[0]]))
        _pin(feats[0][0].cpu().numpy(), *R.truth(R.image_pixels(base[j], K), cs, K, VARIANT), f"base {j} scale 1")
    alone = torch.stack(alone)
    L = alone.shape[1]
    idx = torch.arange(nf, device="cuda") % P
    frames = torch.from_numpy(base).cuda()[idx].contiguous()
    (feats, _), n = _launches(sd, lambda: sd.vl_hog_pyramid(frames, scales, cs, K, VARIANT))
    first, last = feats[0][0], feats[-1][-1]
    assert last.data_ptr() + last.numel() * 4 == first.data_ptr() + nf * L * 4    # the levels lie end to end in slot order
    got = first.as_strided((nf, L), (L, 1), first.storage_offset())
    ok = torch.equal(_bits(got), _bits(alone)[idx])
    print(f"sd_hog_pyramid: {nf * len(scales)} levels, {n} launches (one resize, two dense), every level equals its frame alone: {ok}")
    assert ok
    assert n == 3


def _grids(rng, shapes, dd):
    return [torch.from_numpy(rng.uniform(0, 0.4, (dd, h, w)).astype(np.float32)).cuda() for h, w in shapes]


def _relayout(sd, g, flip, transpose, out):
    ctx = sd.default_context()
    return _capi.lib().sd_hog_relayout(ctx.h, C.byref(g), K, VARIANT, flip, transpose, _capi.ptr(out))


def _batch_grids(t):
    g = HogGridsC()
    g.d_features, g.count, g.height, g.width, g.d_grids = t.data_ptr(), t.shape[0], t.shape[2], t.shape[3], None
    return g


@pytest.mark.parametrize("flip,transpose", [(1, 0), (0, 1), (1, 1)])
def test_relayout_equal_grids_chunks(sd, flip, transpose):
    dd = 3 * K + 4
    base = torch.stack(_grids(np.random.default_rng(7 + 2 * flip + transpose), [(3, 5)] * P, dd))
    alone = []
    for j in range(P):
        o = torch.empty_like(base[j:j + 1])
        assert _relayout(sd, _batch_grids(base[j:j + 1]), flip, transpose, o) == 0
        alone.append(o[0])
    alone = torch.stack(alone)
    if flip and not transpose:
        perm = torch.from_numpy(sd.vl_hog_permutation(VARIANT, K)).cuda()
        assert _same(alone, torch.flip(base[:, perm], dims=[3]))
    grids, idx = _periodic(base)
    n_item = dd * 15
    out = torch.full((11 + N * n_item + 13,), CANARY, dtype=torch.float32, device="cuda")
    rc, n = _launches(sd, lambda: _relayout(sd, _batch_grids(grids), flip, transpose, out[11:]))
    assert rc == 0
    _check_chunked(f"sd_hog_relayout flip {flip} transpose {transpose}", out[11:11 + N * n_item].view(N, -1),
                   alone.reshape(P, -1), idx, n)
    assert bool((out[:11] == CANARY).all()) and bool((out[11 + N * n_item:] == CANARY).all())


@pytest.mark.parametrize("flip,transpose", [(1, 0), (0, 1)])
def test_relayout_grid_table_chunks(sd, flip, transpose):
    dd = 3 * K + 4
    shapes = [(3, 5) if j % 2 == 0 else (2, 7) for j in range(P)]
    base = _grids(np.random.default_rng(30 + flip), shapes, dd)
    feat = torch.cat([b.reshape(-1) for b in base])
    starts = np.cumsum([0] + [b.numel() for b in base])[:-1]
    alone = []
    for j in range(P):
        o = torch.empty_like(base[j][None])
        assert _relayout(sd, _batch_grids(base[j][None]), flip, transpose, o) == 0
        alone.append(o[0])
    sizes = [a.numel() for a in alone]
    j_of = np.arange(N) % P
    offsets = np.cumsum([5] + [sizes[j] + 3 for j in j_of])
    table = (HogGridC * N)(*[HogGridC(shapes[j][1], shapes[j][0], int(starts[j]), int(offsets[i])) for i, j in enumerate(j_of)])
    d_table = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    g = HogGridsC()
    g.d_features, g.count, g.width, g.height, g.d_grids = feat.data_ptr(), N, 0, 0, d_table.data_ptr()
    out = torch.full((int(offsets[-1]) + 7,), CANARY, dtype=torch.float32, device="cuda")
    rc, n = _launches(sd, lambda: _relayout(sd, g, flip, transpose, out))
    assert rc == 0
    _scattered(out, torch.from_numpy(offsets[:-1].astype(np.int64)).cuda(), sizes, torch.from_numpy(j_of).cuda(), alone)
    print(f"sd_hog_relayout table flip {flip} transpose {transpose}: {N} grids, {n} launches, every grid equals its base grid alone")
    assert n == 2


@pytest.mark.parametrize("h,w", [(1, 1), (1, 2)])
def test_render_chunks(sd, h, w):
    dd = 3 * K + 4
    base = torch.stack(_grids(np.random.default_rng(50 + w), [(h, w)] * P, dd))
    alone = torch.cat([sd.vl_hog_render(base[j:j + 1], K, VARIANT) for j in range(P)])
    grids, idx = _periodic(base)
    got, n = _launches(sd, lambda: sd.vl_hog_render(grids, K, VARIANT))
    _check_chunked(f"sd_hog_render {w} x {h} cells", got, alone, idx, n)


# ---- pyramid slices --------------------------------------------------------------------------------------------------------
PYR_CS = 8


def _frame(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = 127.5 + 90 * np.sin(x / 13.0 + np.cos(y / 17.0)) * np.cos(y / 9.0) + rng.normal(0, 12, (h, w))
    return np.clip(np.round(img), 0, 255).astype(np.uint8)


def _pyramid_slices(sd, sizes, scales):
    """The slice rule of sd_hog_pyramid: whole frames while their non-empty levels (rows padded to 16 bytes) fit
    PYRAMID_SLICE_BYTES, one frame at least.  -> (first frame of every slice, level bytes of every slice, launches)."""
    starts, used, launches = [], [], 0
    for f, (h, w) in enumerate(sizes):
        b, nl = 0, 0
        for s in scales:
            (lw, lh), (_, _, hw) = sd.hog_pyramid_shape(w, h, s, PYR_CS, K, VARIANT)
            if hw:
                b += (lw + 15) // 16 * 16 * lh
                nl += 1
        assert nl > 0
        if not starts or used[-1] + b > PYRAMID_SLICE_BYTES:
            starts.append(f)
            used.append(0)
            launches += 2                                        # one resize, one dense launch: far fewer than 65,535 levels
        used[-1] += b
    return starts, used, launches


def _check_pyramid(sd, oracle, frames, batch, scales, what):
    """A fresh context, so that its pyramid scratch starts empty and grows wherever a slice needs more than the last."""
    sizes = [f.shape for f in frames]
    starts, used, expect = _pyramid_slices(sd, sizes, scales)
    ctx = sd.Context()
    _, upload = _launches(sd, lambda: sd._grey_frames(batch, ctx, lambda w, h: None), ctx)
    (feats, lsizes), n = _launches(sd, lambda: sd.vl_hog_pyramid(batch, scales, PYR_CS, K, VARIANT, ctx=ctx), ctx)
    ctx.close()
    n -= upload
    print(f"{what}: {len(frames)} frames, {len(starts)} slices starting at frames {starts}, MB per slice "
          f"{[round(u / 2 ** 20, 1) for u in used]}, {n} launches")
    assert n == expect and len(starts) >= 3
    empty = 0
    for f, fr in enumerate(frames):
        ref, _ = sd.vl_hog_pyramid([fr], scales, PYR_CS, K, VARIANT)
        for s in range(len(scales)):
            if ref[0][s] is None:
                assert feats[f][s] is None
                empty += 1
            else:
                assert _same(feats[f][s], ref[0][s]), (what, f, s)
    edges = sorted({f for s in starts[1:] for f in (s - 1, s)})
    for f in edges:
        for s in range(len(scales)):
            if feats[f][s] is None:
                continue
            lw, lh = lsizes[f][s]
            lvl = frames[f] if (lw, lh) == (frames[f].shape[1], frames[f].shape[0]) else oracle.resize_linear_u8(frames[f], lw, lh)
            assert _same(feats[f][s], sd.hog_dense(torch.from_numpy(lvl)[None].cuda(), PYR_CS, K, VARIANT)[0]), (what, f, s)
    return starts, used, empty


def test_pyramid_several_slices_with_growing_scratch(sd, oracle):
    """Slice 0 stops short because the next frame is large, so slice 1 needs more scratch than slice 0 did."""
    scales = [2.0 * 2 ** (-l / 5) for l in range(25)]
    sizes = [(480, 640)] * 10 + [(1080, 1920), (720, 1280), (480, 640), (480, 640), (1080, 1920), (37, 53)]
    frames = [_frame(h, w, 200 + i) for i, (h, w) in enumerate(sizes)]
    starts, used, empty = _check_pyramid(sd, oracle, frames, frames, scales, "several slices")
    assert used[1] > used[0] and empty > 0


def test_pyramid_frame_larger_than_a_slice(sd, oracle):
    scales = [4.0, 1.0, 0.5]
    frames = [_frame(480, 640, 300), _frame(2000, 2100, 301), _frame(360, 500, 302)]
    starts, used, _ = _check_pyramid(sd, oracle, frames, frames, scales, "a frame larger than a slice")
    assert starts == [0, 1, 2] and used[1] > PYRAMID_SLICE_BYTES


def test_pyramid_slices_of_equally_sized_frames(sd, oracle):
    scales = [2.0 * 2 ** (-l / 5) for l in range(20)]
    frames = [_frame(480, 640, 400 + i) for i in range(30)]
    batch = torch.from_numpy(np.stack(frames)).cuda()
    _check_pyramid(sd, oracle, frames, batch, scales, "equally sized frames")


# ---- trainer slices ----------------------------------------------------------------------------------------------------------
CELL, SIDE = 8, 6


def _train_slices(sd, sizes, scales):
    """The slice rule of sd_hog_train_filter: whole frames while their features fit TRAIN_SLICE_FLOATS, one frame at least"""
    starts, acc = [], 0
    for f, (h, w) in enumerate(sizes):
        fl = 0
        for s in scales:
            _, (dd, hh, hw) = sd.hog_pyramid_shape(w, h, s, CELL, K, VARIANT)
            fl += dd * hh * hw
        if not starts or acc + fl > TRAIN_SLICE_FLOATS:
            starts.append(f)
            acc = 0
        acc += fl
    return starts


def _table_batch(frames):
    """The frames on the device in reverse order with a gap after each, and an ImageBatchC with one descriptor per frame"""
    n, h, w = frames.shape
    stride = h * w + 48
    buf = torch.zeros(n * stride, dtype=torch.uint8)
    for f in range(n):
        o = (n - 1 - f) * stride
        buf[o:o + h * w] = torch.from_numpy(frames[f].ravel())
    buf = buf.cuda()
    table = (FrameC * n)(*[FrameC(w, h, w, 0, (n - 1 - f) * stride) for f in range(n)])
    d_table = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    ib = ImageBatchC(C.c_void_p(buf.data_ptr()), 0, 0, 0, 0, n)
    ib.d_frames = d_table.data_ptr()
    return (buf, d_table), ib


def test_trainer_slices(sd, monkeypatch):
    W, H, n = 320, 240, 64
    frames, boxes = T.planted_frames(2718, n, W, H, sides=(48, 120))
    scales = [4 * 2 ** (-l / 5) for l in range(40) if min(W, H) * 4 * 2 ** (-l / 5) >= CELL * (SIDE + 1)]
    starts = _train_slices(sd, [(H, W)] * n, scales)
    assert len(starts) >= 3
    ends = starts[1:] + [n]
    # boxes in the first and last frame of every slice but slice 1, which has none; a few in between
    box_frame = sorted({f for i, (a, b) in enumerate(zip(starts, ends)) if i != 1 for f in (a, a + 3, b - 2, b - 1)})
    kw = dict(lam=0.01, flip_positives=True, rounds=3, negatives_per_frame=8, mine_overlap=0.5, max_negatives=300)
    args = (box_frame, boxes[box_frame], scales, (SIDE, SIDE), CELL, K)
    on_device = sd.train_hog_filter(torch.from_numpy(frames).cuda(), *args, **kw)
    keep, ib = _table_batch(frames)
    # equally sized host frames are uploaded as one batch without a table, so the table is handed to the trainer directly
    monkeypatch.setattr(sd, "_grey_frames", lambda frames_, ctx, check: (keep, ib, [(H, W)] * n))
    on_table = sd.train_hog_filter(frames, *args, **kw)
    monkeypatch.undo()
    filt, bias, neg, reps = T.train_rule(sd, frames, *args, **kw)
    print(f"trainer: {n} frames, {len(scales)} scales, slices start at {starts}, boxes in frames {box_frame}")
    for r in reps:
        print({k: r[k] for k in T.COUNTS})
    for what, hf in (("device batch", on_device), ("frame table", on_table)):
        assert np.array_equal(hf.filter.cpu().numpy().ravel().view(np.uint32), filt.view(np.uint32)), what
        assert np.float32(hf.bias) == bias, what
        assert np.array_equal(hf.negatives, neg), what
        got = [{k: r[k] for k in T.COUNTS + ("solve",)} for r in hf.report]
        assert got[:len(reps)] == reps, what
    assert sum(r["truncated"] for r in reps) > 0 and sum(r["evicted"] for r in reps) > 0
    slice_of = np.searchsorted(starts, neg[:, 0], side="right") - 1
    assert set(slice_of.tolist()) == set(range(len(starts)))        # negatives from every slice
