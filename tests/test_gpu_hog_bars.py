"""The HOG kernels against the float64 truth of tests/hog_ref64.py, per feature: |kernel - truth| <= bar for every feature, and
exact zeros where the truth and its bar are 0.  The truth takes the kernels' discrete decisions as inputs: the landmark path's
resized patches come from sd_hog_debug (pinned to cv::resize by test_gpu_hog_packed.py) and its bins must equal the oracle's;
float frames and polar fields are built so that every decision keeps a float64 margin (hog_ref64.decided_float_frame,
polar_field).  The inputs put small features next to large ones (a strong edge beside +-1 grey-level texture), flat cells
(exact zeros) and edges that clamp many block sums at 0.2; each case asserts that it reached those cells.

Routes: sd_hog_batch (hog_patch_kernel + hog_normalise_kernel) at every compiled schedule and the run-time ones, both variants,
adaptive and fixed-patch, batches that are not a multiple of the normalise kernel's patches per CTA, odd ld; sd_hog_dense on its
TMA route and its load loop (frame table, odd pitch) at tile edges and sub-cell remainders; sd_hog_dense_images on float and
8-bit frames of 1, 3 (planar and interleaved) and 16 channels, nearest and bilinear; sd_hog_dense_polar, directed and
undirected, nearest and bilinear."""
import ctypes as C
from collections import defaultdict

import numpy as np
import pytest

import hog_ref64 as R
from test_gpu_hog_configs import CONFIGS, L, Layout, _eyes, _param, _sample, device_batch, kernel_of

pytestmark = pytest.mark.gpu
WORST = defaultdict(float)        # (route, variant) -> worst error / bar
WIDTH = defaultdict(list)         # (route, variant) -> bar / |truth| of every non-zero feature


def _record(route, variant, got, want, bar, what):
    r = R.worst(got, want, bar)
    WORST[(route, variant)] = max(WORST[(route, variant)], r)
    nz = want != 0
    WIDTH[(route, variant)].append((bar[nz] / np.abs(want[nz])).astype(np.float32))
    assert got.shape == want.shape, what
    assert r <= 1.0, f"{what}: error / bar {r:.3g}"
    flat = (want == 0) & (bar == 0)
    assert np.all(got[flat] == 0), f"{what}: a feature of a cell without votes is not exactly 0"
    return r


def _reached(kinds, what, flat=True, small=True):
    """The inputs reached clamped block sums, and (where the frames hold enough cells) small features and flat cells."""
    assert kinds["hcf"] > 0, (what, kinds)
    assert kinds["small"] > 0 or not small, (what, kinds)
    assert kinds["flat"] > 0 or not flat, (what, kinds)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nper route and variant: worst error / bar; width of the bar in units of 2^-24 |truth| (median, 99th percentile)")
    for (route, variant), r in sorted(WORST.items()):
        w = np.concatenate(WIDTH[(route, variant)]) / R.U
        print(f"  {route:<28} variant {variant}: {r:.3f}   bar {np.median(w):8.1f} u  {np.percentile(w, 99):8.1f} u")


# ---- landmark path ---------------------------------------------------------------------------------------------------------
FW, FH = 400, 320


def _landmark_frames():
    return [R.blind_spot_frame(FH, FW, seed=s, cs=8) for s in (3, 4)]


def _landmark_samples(fs, n, nl=L):
    """n samples of windows over the frames' edge band, flat block, bright square and texture, and over the frame's corner
    (zero padding: flat).  nl = 3 keeps landmark 2 only (eyes 0 and 1 as with L = 4)."""
    rng = np.random.default_rng(fs + n)
    out = []
    for i in range(n):
        P = int((fs, fs + (fs & 1), 2 * fs, max(2, (2 * fs // 3) & ~1))[i % 4])
        spots = [(0, FH // 5 - P // 2), (FW - P - 2, FH - P - 2), (FW - 3 * FW // 8, 2), (FW // 2, FH // 2), (-(P // 3), -(P // 4))]
        a, b = spots[i % 5], spots[(i + 2) % 5]
        a = (a[0] + int(rng.integers(0, 5)), a[1] + int(rng.integers(0, 5)))
        f, row = _sample(i % 2, P, a, b)
        if nl == 3:
            row = np.concatenate([row[:3], row[L:L + 3]]).astype(np.float32)
        out.append((f, row))
    return out


def _run_landmark(ctx, ib, samples, cfg, fixed, L=L):
    import torch
    from superviseddescent_b200 import _capi
    lib = _capi.lib()
    fs = cfg[1] * cfg[2]
    N = len(samples)
    x = torch.from_numpy(np.stack([r for _, r in samples])).cuda()
    idx = torch.tensor([f for f, _ in samples], dtype=torch.int32, device="cuda")
    p = _param(cfg)
    eyes = None if fixed else C.byref(_eyes())
    geo = torch.empty((N, L, 3), dtype=torch.int32, device="cuda")
    patches = torch.empty((N, L, fs, fs), dtype=torch.uint8, device="cuda")
    bins = torch.empty((N, L, fs, fs), dtype=torch.int8, device="cuda")
    rc = lib.sd_hog_debug(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, eyes, C.byref(p),
                          _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
    assert rc == 0, lib.sd_last_error(ctx.h)
    D = lib.sd_hog_feature_length(L, C.byref(p))
    ld = D + (2 if D % 2 else 1)                                       # an odd ld, past the row
    A = torch.full((N, ld), float("nan"), dtype=torch.float32, device="cuda")
    rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, eyes, C.byref(p),
                          _capi.ptr(A), C.c_int64(ld))
    assert rc == 0, lib.sd_last_error(ctx.h)
    assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
    return patches.cpu().numpy(), bins.cpu().numpy().astype(np.int32), A.cpu().numpy(), D


def _landmark_case(sd, oracle, ctx, ib, cfg, fixed):
    variant, nc, cs, K = cfg
    fs, cells = nc * cs, nc * nc
    # N * L patches, not a multiple of hog_normalise_kernel's patches per CTA, so that its last CTA is partial: where that
    # count divides 4, three landmarks per sample (at 256 / cells = 1 every CTA holds one patch and none is partial)
    per_cta = max(1, 256 // cells)
    L = 3 if per_cta > 1 and 4 % per_cta == 0 else 4
    N = 13
    while per_cta > 1 and (N * L) % per_cta == 0:
        N += 1
    samples = _landmark_samples(fs, N, L)
    patches, bins, A, D = _run_landmark(ctx, ib, samples, cfg, fixed, L)
    ld = A.shape[1]
    assert ld % 2 == 1
    assert np.all(np.isnan(A[:, D:])), "columns past the row were written"
    dd = R.dims(variant, K)
    per_lm = cells * dd
    want = np.zeros((N, D)); bar = np.zeros((N, D))
    tot = defaultdict(int)
    for i in range(N):
        for l in range(L):
            patch = patches[i, l]
            assert np.array_equal(bins[i, l], oracle.hog_orientation_bins(patch.astype(np.float32), K))
            px = R.image_pixels(patch, K)
            st = {}
            f, e = R.truth(px, cs, K, variant, st)
            for k, v in R.kinds(f, e, st).items():
                tot[k] += v
            # row layout [dim][cell col][cell row]
            want[i, l * per_lm:(l + 1) * per_lm] = f.transpose(0, 2, 1).ravel()
            bar[i, l * per_lm:(l + 1) * per_lm] = e.transpose(0, 2, 1).ravel()
    got = A[:, :D]
    n = D - 1                                                         # the features; the fixed-patch functor has no bias
    if not fixed:
        assert np.all(got[:, -1] == 1.0), "bias is not exactly 1"
    route = "landmark " + ("compiled" if kernel_of(cfg)[1] else "run-time") + (" fixed" if fixed else "")
    r = _record(route, variant, got[:, :n], want[:, :n], bar[:, :n], f"{cfg} fixed={fixed}")
    _reached(tot, (cfg, fixed), flat=nc >= 3, small=nc >= 3 and K > 1 and cs > 1)
    return r


@pytest.mark.parametrize("cfg", CONFIGS, ids=[f"v{c[0]}-nc{c[1]}-cs{c[2]}-K{c[3]}" for c in CONFIGS])
def test_landmark_features_within_bars(sd, oracle, cfg):
    """sd_hog_batch at every schedule of CONFIGS, in both variants, adaptive and (even cell sizes) fixed-patch."""
    ctx = sd.default_context()
    ib, keep, _ = device_batch(Layout("tma", _landmark_frames()))
    for variant in (0, 1):
        c = (variant,) + tuple(cfg[1:])
        r = _landmark_case(sd, oracle, ctx, ib, c, fixed=False)
        line = f"{c} kernel {kernel_of(c)} adaptive {r:.3f}"
        if c[2] % 2 == 0:
            r = _landmark_case(sd, oracle, ctx, ib, c, fixed=True)
            line += f" fixed {r:.3f}"
        print(line)


# ---- dense 8-bit grey ------------------------------------------------------------------------------------------------------
def dense_tile(cs):
    """csrc/sd_hog_dense.cu's dense_tile."""
    return max(1, min(14, (112 - 2) // cs - 4))


def _extent(g, cs, past):
    """Pixels of a frame side with g cells: W mod cs = cs / 2 - 1 (the cells end inside the frame), or with the last cell
    reaching past the frame ((g - 1) cs + ceil(cs / 2) pixels)."""
    if cs == 1:
        return g
    return (g - 1) * cs + (cs + 1) // 2 if past else g * cs + cs // 2 - 1


def dense_sizes(cs):
    """(H, W) whose hogW sits at 2 tile - 1, 2 tile and 2 tile + 1 and hogH at tile, tile + 1 and 2 tile (dense_tile's tile),
    alternating the two remainders of _extent."""
    T = dense_tile(cs)
    out = []
    for j, (gw, gh) in enumerate(zip((2 * T - 1, 2 * T, 2 * T + 1), (T, T + 1, 2 * T))):
        W, H = _extent(gw, cs, j % 2 == 1), _extent(gh, cs, j % 2 == 0)
        if min(W, H) < 4:
            continue
        assert R.grid(W, H, cs) == (gw, gh), (cs, W, H)
        out.append((H, W))
    return out


DENSE_CS = list(range(1, 13)) + [13, 16, 17, 20, 24, 31, 32]


@pytest.mark.parametrize("cs", DENSE_CS)
def test_dense_u8_features_within_bars(sd, oracle, cs):
    """sd_hog_dense at tile edges: the TMA route (one device batch, 16-byte pitch), the load loop through an odd pitch, and the
    frame table (frames of several sizes, 4 x 4 and 7 x 5 among them)."""
    import torch
    K = (1, 4, 9, 16)[cs % 4]
    sizes = dense_sizes(cs)
    tot = defaultdict(int)
    for variant in (0, 1):
        frames = [R.blind_spot_frame(H, W, seed=cs * 7 + H + variant, cs=cs) for H, W in sizes]
        for (H, W), f in zip(sizes, frames):
            for pitch in ((W + 15) // 16 * 16, W + 1 + (W % 2 == 0)):
                big = torch.zeros((2, H, pitch), dtype=torch.uint8)
                big[0, :, :W] = torch.from_numpy(f)
                big[1, :, :W] = torch.from_numpy(f[::-1].copy())
                dev = big.cuda()[:, :, :W]
                got = sd.hog_dense(dev, cs, K, variant).cpu().numpy()
                for i, img in enumerate((f, f[::-1].copy())):
                    st = {}
                    want, bar = R.truth(R.image_pixels(img, K), cs, K, variant, st)
                    for k, v in R.kinds(want, bar, st).items():
                        tot[k] += v
                    route = "dense u8 tma" if pitch % 16 == 0 else "dense u8 odd pitch"
                    _record(route, variant, got[i], want, bar, f"cs {cs} K {K} {W} x {H} pitch {pitch}")
        extra = [R.blind_spot_frame(4, 4, seed=1, cs=1), R.blind_spot_frame(5, 7, seed=2, cs=1)] if cs <= 4 else []
        table = frames + extra
        got = sd.hog_dense(table, cs, K, variant)
        for g, img in zip(got, table):
            want, bar = R.truth(R.image_pixels(img, K), cs, K, variant)
            _record("dense u8 frame table", variant, g.cpu().numpy(), want, bar, f"cs {cs} K {K} table {img.shape}")
    _reached(tot, cs, flat=cs <= 13, small=cs <= 13)
    print(f"dense u8 cs {cs} K {K}: {dict(tot)}")


# ---- float and multi-channel frames ----------------------------------------------------------------------------------------
IMAGE_CASES = R.IMAGE_CASES


@pytest.mark.parametrize("case", IMAGE_CASES, ids=[f"c{c[0]}-{c[1]}-cs{c[2]}-K{c[3]}" for c in IMAGE_CASES])
@pytest.mark.parametrize("bil", [False, True])
def test_images_features_within_bars(sd, case, bil):
    """sd_hog_dense_images on float frames (values in [0, 255] or [0, 1]) and on 8-bit frames through the same entry."""
    C_, layout, cs, K, H, W, scale = case
    tot = defaultdict(int)
    for kind in ("f32", "u8"):
        f = R.image_case_frame(case, kind, bil)
        batch = f[None] if layout == "planar" else np.ascontiguousarray(np.moveaxis(f, 0, -1))[None]
        for variant in (0, 1):
            got = sd.vl_hog(batch, cs, K, variant, bilinear_orientations=bil, channels_last=layout != "planar").cpu().numpy()[0]
            st = {}
            px = R.image_pixels(f if C_ > 1 else f[0], K, bil, check_margin=kind == "f32")
            want, bar = R.truth(px, cs, K, variant, st)
            for k, v in R.kinds(want, bar, st).items():
                tot[k] += v
            route = f"images {kind}" + (" bilinear" if bil else "")
            _record(route, variant, got, want, bar, f"{case} {kind} bilinear {bil} variant {variant}")
    _reached(tot, case, flat=cs <= 11, small=cs <= 11 and K > 1)


# ---- polar fields ----------------------------------------------------------------------------------------------------------
POLAR_CASES = [(4, 4, 37, 45), (1, 1, 12, 15), (8, 9, 50, 61), (3, 16, 29, 31), (32, 2, 70, 66), (5, 9, 4, 4), (2, 4, 5, 7)]


@pytest.mark.parametrize("case", POLAR_CASES, ids=[f"cs{c[0]}-K{c[1]}-{c[3]}x{c[2]}" for c in POLAR_CASES])
def test_polar_features_within_bars(sd, case):
    """sd_hog_dense_polar: moduli over six orders of magnitude, a zero row and a column of negative moduli (which do not vote),
    every pixel voting including the border."""
    cs, K, H, W = case
    tot = defaultdict(int)
    for directed in (True, False):
        for bil in (False, True):
            m, a = R.polar_field(H, W, seed=cs * 13 + K + H, K=K, directed=directed, bilinear=bil)
            if H > 4 * cs:
                m[: 2 * cs + 2, : 2 * cs + 2] = 0                     # a flat corner
            px = R.polar_pixels(m, a, K, directed, bil)
            assert np.any(px.bins[0][0] >= 0) and np.any(px.bins[0][:, 0] >= 0)   # border pixels vote
            for variant in (0, 1):
                got = sd.vl_hog_polar(m[None], a[None], cs, K, variant, directed=directed,
                                      bilinear_orientations=bil).cpu().numpy()[0]
                st = {}
                want, bar = R.truth(px, cs, K, variant, st)
                for k, v in R.kinds(want, bar, st).items():
                    tot[k] += v
                route = "polar " + ("directed" if directed else "undirected") + (" bilinear" if bil else "")
                _record(route, variant, got, want, bar, f"{case} directed {directed} bilinear {bil} variant {variant}")
    _reached(tot, case, flat=H > 4 * cs, small=H > 4 * cs and K > 1)
