"""HOG filter scores on the device (sd_hog_correlate, api.vl_hog_correlate) against float64 with per-element error bars.

The kernel forms every score as one float32 FMA chain from 0 over the n = dd * fh * fw products (channel, dy, dx ascending; the
zero padding contributes exact zeros), then adds the bias with one rounding.  With u = 2^-24, each FMA rounds once, so the chain
is within gamma_n * sum |F M| of the exact sum (gamma_n = n u / (1 - n u)), and the bias addition adds u |S + bias|.  Hence

    |S - S64| <= tau * sum |F * M| + u |bias|,    tau = (n + 1) u / (1 - (n + 1) u),

where S64 is float64 conv2d on the CPU.  The worst error / bar of every case is printed."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
CANARY = -777.25


def _dd(K, variant):
    return 3 * K + 4 if variant == 1 else 4 * K


def _maps(sizes, dd, seed):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.uniform(0, 0.4, (dd, h, w)).astype(np.float32)).cuda() for h, w in sizes]


def _truth(m, f, bias, pad):
    """(score, bar) in float64 on the CPU."""
    px, py = pad
    q, _, fh, fw = f.shape
    oh, ow = m.shape[1] + 2 * py - fh + 1, m.shape[2] + 2 * px - fw + 1
    if oh <= 0 or ow <= 0:
        z = torch.zeros((q, max(oh, 0), max(ow, 0)), dtype=torch.float64)
        return z, z
    m64, f64 = m.double().cpu()[None], f.double().cpu()
    s = Fn.conv2d(m64, f64, padding=(py, px))[0]
    a = Fn.conv2d(m64.abs(), f64.abs(), padding=(py, px))[0]
    n = f.shape[1] * f.shape[2] * f.shape[3]
    tau = (n + 1) * U / (1 - (n + 1) * U)
    bar = tau * a
    if bias is not None:
        b = bias.double().cpu()[:, None, None]
        s = s + b
        bar = bar + U * b.abs()
    return s, bar


def _check(got, m, f, bias, pad, label):
    s, bar = _truth(m, f, bias, pad)
    assert tuple(got.shape) == tuple(s.shape), (label, got.shape, s.shape)
    if s.numel() == 0:
        return 0.0
    err = (got.double().cpu() - s).abs()
    ratio = float((err / bar.clamp_min(1e-300)).max())
    print(f"{label}: worst error / bar {ratio:.3f}")
    assert bool((err <= bar).all()), (label, ratio)
    return ratio


CASES = [
    # K, variant, (fh, fw), Q, pad (x, y), grid sizes (h, w)
    (9, 1, (6, 6), 1, (0, 0), [(90, 160), (1, 1), (16, 32), (21, 37), (22, 38), (17, 33), (6, 6), (5, 9)]),
    (9, 1, (6, 6), 2, (5, 5), [(1, 1), (15, 31), (40, 70)]),
    (4, 1, (1, 1), 9, (0, 0), [(3, 5), (16, 32), (33, 65)]),
    (16, 0, (3, 7), 8, (3, 1), [(12, 40), (2, 2), (31, 47)]),
    (4, 0, (8, 5), 3, (2, 4), [(20, 19), (8, 5)]),
    (16, 1, (2, 9), 4, (8, 0), [(9, 50), (1, 3)]),
    (9, 0, (32, 32), 1, (31, 0), [(40, 35), (1, 1)]),
    (4, 1, (32, 17), 5, (10, 20), [(33, 18)]),
    (9, 1, (6, 6), 256, (2, 3), [(20, 30), (5, 5)]),
    (4, 0, (4, 4), 17, (1, 1), [(18, 34)]),
]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("with_bias", [True, False])
def test_scores_within_bars(sd, case, with_bias):
    K, variant, (fh, fw), Q, pad, sizes = CASES[case]
    dd = _dd(K, variant)
    rng = np.random.default_rng(100 + case)
    f = torch.from_numpy(rng.normal(0, 1, (Q, dd, fh, fw)).astype(np.float32)).cuda()
    bias = torch.from_numpy(rng.normal(0, 3, Q).astype(np.float32)).cuda() if with_bias else None
    maps = _maps(sizes, dd, case)
    got = sd.vl_hog_correlate(maps, f, K, variant, bias=bias, pad=pad)
    for i, (m, g) in enumerate(zip(maps, got)):
        _check(g, m, f, bias, pad, f"case {case} grid {i} {tuple(m.shape)}")


def test_real_hog_pyramid_in_place(sd):
    """Pyramid levels (views of one buffer) are scored in place, including levels smaller than the filter."""
    rng = np.random.default_rng(3)
    y, x = np.mgrid[0:200, 0:260]
    img = np.clip(128 + 80 * np.sin(x / 9.0) * np.cos(y / 14.0) + rng.normal(0, 10, (200, 260)), 0, 255).astype(np.uint8)
    scales = [2 ** (-l / 5) for l in range(0, 25)]
    feats, _ = sd.vl_hog_pyramid([img], scales, 8, 9, 1)
    levels = [v for v in feats[0] if v is not None]
    assert len({v.untyped_storage().data_ptr() for v in levels}) == 1
    f = torch.from_numpy(rng.normal(0, 1, (2, 31, 6, 6)).astype(np.float32)).cuda()
    got = sd.vl_hog_correlate(levels, f, 9, 1)
    assert any(g.numel() == 0 for g in got)
    for m, g in zip(levels, got):
        _check(g, m, f, None, (0, 0), f"level {tuple(m.shape)}")


def test_grid_alone_equals_grid_in_batch(sd):
    K, variant = 9, 1
    maps = _maps([(45, 80), (7, 9), (90, 160), (1, 1), (33, 65)], 31, 8)
    f = torch.from_numpy(np.random.default_rng(9).normal(0, 1, (9, 31, 6, 6)).astype(np.float32)).cuda()
    bias = torch.arange(9, dtype=torch.float32, device="cuda") * 0.1
    batch = sd.vl_hog_correlate(maps, f, K, variant, bias=bias, pad=(2, 3))
    for m, b in zip(maps, batch):
        alone = sd.vl_hog_correlate([m], f, K, variant, bias=bias, pad=(2, 3))[0]
        assert torch.equal(alone, b)
    # one filter of the bank alone gives its own rows bit for bit
    one = sd.vl_hog_correlate(maps, f[4:5].contiguous(), K, variant, bias=bias[4:5].contiguous(), pad=(2, 3))
    for o, b in zip(one, batch):
        assert torch.equal(o[0], b[4])


@pytest.mark.parametrize("K,variant", [(9, 1), (4, 0)])
def test_flip_gives_mirrored_scores(sd, K, variant):
    dd = _dd(K, variant)
    maps = _maps([(30, 47)], dd, 12)
    f = torch.from_numpy(np.random.default_rng(13).normal(0, 1, (2, dd, 5, 7)).astype(np.float32)).cuda()
    pad = (3, 2)
    s = sd.vl_hog_correlate(maps, f, K, variant, pad=pad)[0]
    mf = sd.vl_hog_flip(maps, K, variant)
    ff = sd.vl_hog_flip(f, K, variant)
    sf = sd.vl_hog_correlate(mf, ff, K, variant, pad=pad)[0]
    _check(torch.flip(sf, dims=[2]), maps[0], f, None, pad, "mirrored")
    _check(s, maps[0], f, None, pad, "direct")


def test_descriptor_gaps_keep_canaries(sd):
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import HogGridC, HogGridsC
    K, variant, dd, Q, fh, fw = 9, 1, 31, 3, 4, 6
    sizes = [(20, 25), (2, 3), (16, 32), (9, 6)]
    rng = np.random.default_rng(21)
    feat = torch.from_numpy(rng.uniform(0, 0.4, 5000 * dd).astype(np.float32)).cuda()
    f = torch.from_numpy(rng.normal(0, 1, (Q, dd, fh, fw)).astype(np.float32)).cuda()
    descs, pos_in, pos_out, spans = [], 11, 7, []
    for h, w in sizes:
        oh, ow = h - fh + 1, w - fw + 1
        descs.append(HogGridC(w, h, pos_in, pos_out if oh > 0 and ow > 0 else 0))
        if oh > 0 and ow > 0:
            spans.append((pos_in, h, w, pos_out, oh, ow))
            pos_out += Q * oh * ow + 13
        pos_in += dd * h * w + 5
    table = (HogGridC * len(descs))(*descs)
    d_table = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    g = HogGridsC()
    g.d_features, g.count, g.width, g.height, g.d_grids = feat.data_ptr(), len(descs), 0, 0, d_table.data_ptr()
    out = torch.full((pos_out + 40,), CANARY, dtype=torch.float32, device="cuda")
    ctx = sd.default_context()
    assert _capi.lib().sd_hog_correlate(ctx.h, C.byref(g), K, variant, _capi.ptr(f), Q, fw, fh, None, 0, 0, _capi.ptr(out)) == 0
    torch.cuda.synchronize()
    mask = torch.ones_like(out, dtype=torch.bool)
    for pi, h, w, po, oh, ow in spans:
        m = feat[pi:pi + dd * h * w].view(dd, h, w)
        _check(out[po:po + Q * oh * ow].view(Q, oh, ow), m, f, None, (0, 0), f"gap grid {h}x{w}")
        mask[po:po + Q * oh * ow] = False
    assert bool((out[mask] == CANARY).all())
    assert len(spans) == 3


@pytest.mark.parametrize("Q", [1, 2, 3, 9, 256])
def test_equally_sized_grids_without_a_table(sd, Q):
    """A batch tensor of grids with d_grids = NULL: grid i's scores at d_scores + i Q oh ow, within the bars and bit for bit the
    scores of the same maps passed with a table; one call per grid size (the route has one size per call)."""
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import HogGridsC
    K, variant, fh, fw, count, lead, tail = 9, 1, 6, 6, 3, 13, 29
    dd = _dd(K, variant)
    rng = np.random.default_rng(300 + Q)
    f = torch.from_numpy(rng.normal(0, 1, (Q, dd, fh, fw)).astype(np.float32)).cuda()
    bias = torch.from_numpy(rng.normal(0, 3, Q).astype(np.float32)).cuda()
    ctx = sd.default_context()
    # partial tiles in both directions, a 1 x 1 grid (scored through the pads), and a grid smaller than the filter
    for (h, w), pad in [((33, 65), (0, 0)), ((17, 31), (2, 3)), ((1, 1), (5, 5)), ((4, 5), (0, 0))]:
        batch = torch.from_numpy(rng.uniform(0, 0.4, (count, dd, h, w)).astype(np.float32)).cuda()
        oh, ow = h + 2 * pad[1] - fh + 1, w + 2 * pad[0] - fw + 1
        n = Q * max(oh, 0) * max(ow, 0)
        out = torch.full((lead + count * n + tail,), CANARY, dtype=torch.float32, device="cuda")
        g = HogGridsC()
        g.d_features, g.count, g.width, g.height, g.d_grids = batch.data_ptr(), count, w, h, None
        rc = _capi.lib().sd_hog_correlate(ctx.h, C.byref(g), K, variant, _capi.ptr(f), Q, fw, fh, _capi.ptr(bias), pad[0], pad[1],
                                          _capi.ptr(out[lead:]))
        assert rc == 0
        torch.cuda.synchronize()
        assert bool((out[:lead] == CANARY).all()) and bool((out[lead + count * n:] == CANARY).all()), (h, w)
        if n == 0:
            print(f"Q {Q} grid {h}x{w}: smaller than the filter, nothing written")
            continue
        got = out[lead:lead + count * n].view(count, Q, oh, ow)
        table = sd.vl_hog_correlate(list(batch), f, K, variant, bias=bias, pad=pad)
        for i in range(count):
            _check(got[i], batch[i], f, bias, pad, f"Q {Q} equally sized grid {i} {h}x{w} pad {pad}")
            assert torch.equal(got[i].view(torch.int32), table[i].view(torch.int32)), (Q, h, w, i)


def test_refusals_leave_scores_untouched(sd):
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import HogGridsC
    lib = _capi.lib()
    ctx = sd.default_context()
    feat = torch.rand(31 * 10 * 10 + 1, device="cuda")
    f = torch.rand(64 * 31 * 33 * 33 + 1, device="cuda")
    out = torch.full((100000,), CANARY, dtype=torch.float32, device="cuda")
    g = HogGridsC()
    g.d_features, g.count, g.width, g.height, g.d_grids = feat.data_ptr(), 1, 10, 10, None
    P = _capi.ptr
    odd = C.c_void_p(f.data_ptr() + 2)
    bad = [
        (9, 1, P(f), 1, 6, 6, None, 6, 0, P(out)),         # pad_x = fw
        (9, 1, P(f), 1, 6, 6, None, 0, -1, P(out)),        # negative pad
        (9, 1, P(f), 1, 33, 6, None, 0, 0, P(out)),        # fw over the cap
        (9, 1, P(f), 1, 6, 0, None, 0, 0, P(out)),         # fh = 0
        (9, 1, P(f), 0, 6, 6, None, 0, 0, P(out)),         # Q = 0
        (9, 1, P(f), 257, 6, 6, None, 0, 0, P(out)),       # Q over the cap
        (9, 1, None, 1, 6, 6, None, 0, 0, P(out)),         # null filters
        (9, 1, odd, 1, 6, 6, None, 0, 0, P(out)),          # unaligned filters
        (9, 1, P(f), 1, 6, 6, odd, 0, 0, P(out)),          # unaligned bias
        (9, 1, P(f), 1, 6, 6, None, 0, 0, None),           # null scores
        (17, 1, P(f), 1, 6, 6, None, 0, 0, P(out)),        # num_bins
        (9, 2, P(f), 1, 6, 6, None, 0, 0, P(out)),         # variant
    ]
    for args in bad:
        assert lib.sd_hog_correlate(ctx.h, C.byref(g), *args) == 1, args
    assert lib.sd_hog_correlate(ctx.h, None, 9, 1, P(f), 1, 6, 6, None, 0, 0, P(out)) == 1
    # a negative offset in a descriptor
    from superviseddescent_b200._capi import HogGridC
    table = (HogGridC * 1)(HogGridC(10, 10, -1, 0))
    d_table = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    g.d_grids = d_table.data_ptr()
    assert lib.sd_hog_correlate(ctx.h, C.byref(g), 9, 1, P(f), 1, 6, 6, None, 0, 0, P(out)) == 1
    torch.cuda.synchronize()
    assert bool((out == CANARY).all())
