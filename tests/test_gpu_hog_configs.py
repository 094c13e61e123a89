"""The landmark HOG kernel (hog_patch_kernel, csrc/sd_hog.cu) against the oracle at every configuration it accepts and on every
route by which a P x P source window reaches shared memory.

Each sample has L = 4 landmarks, ids "0".."3", right eye "0" and left eye "1".  The eyes sit P px apart on one row at integer
coordinates and relative_patch_size is 1, so the inter-eye distance is exactly P and every window of the sample is P x P
(half = P / 2); landmarks 2 and 3 are placed to pick their windows' x0, y0.  The truth is the oracle's glue (patch_geometry,
crop_patch_u8, resize_linear_u8, pinned to cv2 by tests/golden/resize_cv2*.npz) around the reference's hog.c when oracle/_ref
is built, else around the oracle's restatement of it (pinned bit for bit at these configurations by
test_oracle_hog_core_matches_hog_c_at_every_config).  Geometry, resized patches and orientation bins must be equal, the
features within 1e-5 max-norm relative (the kernel's vote sums in another order than hog.c's raster order).

Batches are built by hand (ImageBatchC with chosen pitches, frame tables and ROIs), so that each window's route is known in
advance from a restatement of hog_smem_layout and of the route rule of hog_patch_kernel's S1:
  tma       a tensor-map box (eight size classes, 32 .. 160) that covers P + (x0 mod 16) and fits the staging area; only for
            batches of whole, equally sized frames with 16-byte aligned base and pitches;
  vec16     16-byte loads: window inside the frame (and ROI), 16-byte aligned base and pitch;
  words     4-byte loads: the same with 4-byte alignment;
  bytes     byte loads with zero padding: any other window that the staging area holds;
  unstaged  resize straight from global memory: ((P + 30) & ~15) * P bytes exceed the staging area.
The same windows of the same frames go through every layout, and their features must be bit-identical across routes.
"""
import ctypes as C
import importlib.util
import os
from collections import Counter

import numpy as np
import pytest

from conftest import rel_err

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_spec = importlib.util.spec_from_file_location("gen_resize_wide", os.path.join(GOLDEN, "gen_resize_wide.py"))
_wide = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_wide)

SMEM_LIMIT = 227 * 1024          # launch_hog's check: the H100's opt-in shared memory per block
TMA_BOXES = (32, 48, 64, 80, 96, 112, 128, 160)
FEATURE_TOL = 1e-5
L = 4
W, H = 400, 320                  # frames of the batches (at least 160 x 160: every TMA box fits inside)
SMALL = (20, 24)                 # (h, w) of a frame smaller than its windows, in the frame-table layout

# (variant, num_cells, cell_size, num_bins): every kernel instantiation the launcher selects, both variants, odd K and cell
# sizes, K = 1, cell size 1, one cell, fs from 4 to 192 across the resize's column-per-thread / warp-per-row switch at 64, and
# the largest layout that fits SMEM_LIMIT for several (num_cells, K)
CONFIGS = [
    (1, 1, 4, 1), (1, 2, 2, 3), (0, 3, 5, 2), (1, 4, 3, 1), (1, 7, 9, 1), (1, 6, 7, 5), (1, 16, 1, 8),
    (1, 5, 8, 9), (0, 5, 10, 9), (1, 5, 11, 9), (1, 5, 6, 9),
    (1, 5, 11, 4), (0, 5, 10, 4), (1, 5, 8, 4), (1, 5, 6, 4),
    (1, 8, 8, 16), (1, 5, 13, 7), (1, 8, 10, 4), (0, 6, 12, 16),
    (1, 12, 6, 16), (1, 16, 9, 4), (1, 5, 33, 9), (1, 5, 36, 4), (1, 1, 192, 4),
]
LARGEST = [(1, 12, 6, 16), (1, 16, 9, 4), (1, 5, 33, 9), (1, 5, 36, 4), (1, 1, 192, 4)]
# the configurations whose routes are enumerated: fs = 4 (no TMA class fits), 30, 55 at K = 4 and 9, and 80
ROUTE_CONFIGS = [(1, 1, 4, 1), (1, 5, 6, 4), (1, 5, 11, 4), (1, 5, 11, 9), (1, 8, 10, 4)]
LAYOUTS = ("tma", "stride", "words", "bytes", "frames", "roi")
ROUTES = ("tma", "vec16", "words", "bytes", "unstaged")


def _align(v, a):
    return (v + a - 1) // a * a


def _dd(variant, K):
    return 3 * K + 4 if variant == 1 else 4 * K


def smem_layout(cfg):
    """hog_smem_layout (csrc/sd_hog.cu) restated: (bytes of the staging area [bin | r1 | vote], total bytes)."""
    variant, nc, cs, K = cfg
    fs, cells = nc * cs, nc * nc
    o = _align(cells * 2 * K * 4, 16)                          # energy
    o = _align(o + cells * 4, 16)                              # fac
    o = max(o + cells * 4 * 8, fs * fs)                        # patch shares with hist / energy / fac
    o = _align(o, 16) + 5 * fs * 4 + nc * fs * 4 + 2 * nc * 4  # resize tables, wcell, lo, hi
    o = _align(_align(o, 8) + 8, 128)                          # mbar
    stage = o
    o = _align(o + fs * fs, 16)                                # bin
    o = _align(o + max(fs * fs * 4, cells * K * 32), 16)       # r1
    o += max(2 * K * _align((fs - 2) * nc, 32) * 4, cells * _dd(variant, K) * 4)
    return o - stage, _align(o, 16)


def accepted(cfg):
    """launch_hog's argument checks."""
    variant, nc, cs, K = cfg
    fs = nc * cs
    return (1 <= K <= 16 and 3 < fs <= 256 and (fs + cs // 2) // cs == nc and smem_layout(cfg)[1] <= SMEM_LIMIT)


def kernel_of(cfg):
    """The hog_patch_kernel<KT, NCT, CST> instantiation launch_hog picks."""
    variant, nc, cs, K = cfg
    if nc == 5 and K in (4, 9) and cs in (11, 10, 8, 6):
        return (K, 5, cs)
    return (K, 0, 0) if K in (4, 9) else (0, 0, 0)


def largest_staged(cap):
    """Largest even window the load loops stage: its (P + 30) & ~15 byte pitch times P rows fits the staging area."""
    return max(P for P in range(2, 2048, 2) if ((P + 30) & ~15) * P <= cap)


def route(cap, P, x0, y0, fr):
    """The route of one window (hog_patch_kernel S1).  fr: tma, W, H, roi (rx, ry, rw, rh), align (address | pitch)."""
    if fr["tma"]:
        for b in TMA_BOXES:
            if b >= P + (x0 & 15) and b * b <= cap:
                return "tma"
    if ((P + 30) & ~15) * P > cap:
        return "unstaged"
    rx, ry, rw, rh = fr["roi"]
    resident = (x0 >= rx and y0 >= ry and x0 + P <= rx + rw and y0 + P <= ry + rh and x0 >= 0 and y0 >= 0
                and x0 + P <= fr["W"] and y0 + P <= fr["H"])
    if resident and fr["align"] % 16 == 0:
        return "vec16"
    if resident and fr["align"] % 4 == 0:
        return "words"
    return "bytes"


# ---- samples -----------------------------------------------------------------------------------------------------------
def _frames():
    """Two W x H frames (noise, and a 5 x 5 box blur of noise) and one SMALL frame of noise."""
    rng = np.random.default_rng(2026)
    f0 = rng.integers(0, 256, (H, W), dtype=np.uint8)
    n = rng.integers(0, 256, (H + 4, W + 4)).astype(np.float64)
    f1 = np.round(np.lib.stride_tricks.sliding_window_view(n, (5, 5)).mean(axis=(2, 3))).astype(np.uint8)
    return [f0, f1, rng.integers(0, 256, SMALL, dtype=np.uint8)]


def _sample(frame, P, a, b, eyes=None):
    """(frame index, landmark row) of a sample whose landmarks 2 and 3 have windows at a = (x0, y0) and b; the eyes P apart,
    centred on the frame unless given."""
    ex, ey = eyes if eyes is not None else (W // 2 - P // 2, H // 2)
    h = P // 2
    row = np.array([ex, ex + P, a[0] + h, b[0] + h, ey, ey, a[1] + h, b[1] + h], dtype=np.float32)
    return frame, row


def _windows_of(row, P):
    h = P // 2
    return [(int(row[l]) - h, int(row[L + l]) - h) for l in range(L)]


def _pairs(frame, wins):
    """Samples holding the windows [(P, x0, y0)] two at a time (landmarks 2 and 3), windows of one P together."""
    out = []
    for P in sorted({w[0] for w in wins}):
        ws = [(x, y) for p, x, y in wins if p == P]
        if len(ws) % 2:
            ws.append(ws[-1])
        out += [_sample(frame, P, ws[i], ws[i + 1]) for i in range(0, len(ws), 2)]
    return out


def route_samples(cfg):
    """Windows that drive each route of this configuration to its edges: every TMA class at P + x0 mod 16 = box and box + 1,
    the largest staged load-loop window and the next even one (unstaged), staged and unstaged windows over every edge and
    corner and wholly outside; on frames 0 and 1.  The frame-table layout adds windows larger than its small frame 2."""
    cap = smem_layout(cfg)[0]
    pst = largest_staged(cap)
    wins = []
    for b in TMA_BOXES:
        if b * b <= cap:
            wins += [(b, 80, 24), (b - 2, 82, 24), (b - 2, 83, 24)]
    wins += [(pst, 64, 8), (pst + 2, 64, 8), (pst + 2, 48, 40)]
    for P in sorted({min(pst, 40), pst + 2}):
        for x0 in (-(P // 3), W // 2 - P // 2, W - 2 * P // 3):
            for y0 in (-(P // 3), H // 2 - P // 2, H - 2 * P // 3):
                wins.append((P, x0, y0))
        wins += [(P, -P - 5, 50), (P, W + 7, 60), (P, 30, H + 3), (P, -P - 20, -P - 9)]
    common = _pairs(0, wins) + _pairs(1, wins[::-1])
    sh, sw = SMALL
    small = [_sample(2, P, (-3, -2), (-(P // 2), -(P // 3)), eyes=(sw // 2 - P // 2, sh // 2)) for P in sorted({30, pst + 2})]
    return common, small


# ---- batches -----------------------------------------------------------------------------------------------------------
class Layout:
    """Where the frames sit in one device buffer: per frame byte offset and pitch (of the ROI for 'roi'), route descriptor."""

    def __init__(self, kind, frames, rois=None):
        self.kind = kind
        self.frames = frames if kind == "frames" else frames[:len(rois) if kind == "roi" else 2]
        n = len(self.frames)
        self.offsets, self.pitches, self.image_stride = [], [], 0
        if kind in ("frames", "roi"):
            o = 0
            for i, f in enumerate(self.frames):
                w, h = (rois[i][2], rois[i][3]) if kind == "roi" else (f.shape[1], f.shape[0])
                self.offsets.append(o)
                self.pitches.append(_align(w, 16))
                o = _align(o + _align(w, 16) * h, 16)
            self.total = o
        else:
            pitch = {"tma": _align(W, 16), "stride": _align(W, 16), "words": _align(W, 16) + 4, "bytes": W + 1}[kind]
            self.image_stride = _align(pitch * H, 16) + (4 if kind == "stride" else 0)
            self.offsets = [i * self.image_stride for i in range(n)]
            self.pitches = [pitch] * n
            self.total = n * self.image_stride
        self.rois = rois
        self.desc = []
        for i, f in enumerate(self.frames):
            roi = tuple(rois[i][:4]) if kind == "roi" else (0, 0, f.shape[1], f.shape[0])
            self.desc.append({"tma": kind == "tma", "W": f.shape[1], "H": f.shape[0], "roi": roi,
                              "align": self.offsets[i] | self.pitches[i]})

    def host_buffer(self):
        buf = np.zeros(self.total, dtype=np.uint8)
        for i, f in enumerate(self.frames):
            if self.kind == "roi":
                rx, ry, rw, rh = self.rois[i]
                f = f[ry:ry + rh, rx:rx + rw]
            h, w = f.shape
            buf[self.offsets[i]:self.offsets[i] + self.pitches[i] * h].reshape(h, self.pitches[i])[:, :w] = f
        return buf


class RoiC(C.Structure):
    """sd_roi."""
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("w", C.c_int32), ("h", C.c_int32), ("row_stride", C.c_int32),
                ("reserved", C.c_int32), ("offset", C.c_int64)]


def _device_table(structs):
    import torch
    raw = b"".join(bytes(s) for s in structs)
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()


def device_batch(lay):
    """(ImageBatchC, tensors to keep alive, d_roi_miss or None) of a Layout."""
    import torch
    from superviseddescent_b200._capi import FrameC, ImageBatchC
    buf = torch.from_numpy(lay.host_buffer()).cuda()
    assert buf.data_ptr() % 16 == 0
    keep = [buf]
    f0 = lay.frames[0]
    ib = ImageBatchC(C.c_void_p(buf.data_ptr()), f0.shape[1], f0.shape[0], lay.pitches[0], lay.image_stride, len(lay.frames))
    miss = None
    if lay.kind == "frames":
        t = _device_table([FrameC(f.shape[1], f.shape[0], lay.pitches[i], 0, lay.offsets[i]) for i, f in enumerate(lay.frames)])
        keep.append(t)
        ib.d_frames = C.c_void_p(t.data_ptr())
    if lay.kind == "roi":
        t = _device_table([RoiC(*r[:4], lay.pitches[i], 0, lay.offsets[i]) for i, r in enumerate(lay.rois)])
        miss = torch.zeros(len(lay.frames), dtype=torch.uint8, device="cuda")
        keep += [t, miss]
        ib.d_roi = C.c_void_p(t.data_ptr())
        ib.d_roi_miss = C.c_void_p(miss.data_ptr())
    return ib, keep, miss


def _param(cfg):
    from superviseddescent_b200._capi import HogParam
    return HogParam(cfg[0], cfg[1], cfg[2], cfg[3], 1.0)


def _eyes():
    from superviseddescent_b200._capi import NormalisationC
    return NormalisationC(1, 1, 1, (C.c_int32 * 4)(0, 0, 0, 0), (C.c_int32 * 4)(1, 0, 0, 0))


def run_kernel(ctx, ib, samples, cfg):
    """sd_hog_debug and sd_hog_batch on the samples: geometry (N, L, 3), patches and bins (N, L, fs, fs), features (N, D)."""
    import torch
    from superviseddescent_b200 import _capi
    lib = _capi.lib()
    fs = cfg[1] * cfg[2]
    N = len(samples)
    x = torch.from_numpy(np.stack([r for _, r in samples])).cuda()
    idx = torch.tensor([f for f, _ in samples], dtype=torch.int32, device="cuda")
    p, eyes = _param(cfg), _eyes()
    geo = torch.empty((N, L, 3), dtype=torch.int32, device="cuda")
    patches = torch.empty((N, L, fs, fs), dtype=torch.uint8, device="cuda")
    bins = torch.empty((N, L, fs, fs), dtype=torch.int8, device="cuda")
    rc = lib.sd_hog_debug(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, C.byref(eyes), C.byref(p),
                          _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
    assert rc == 0, lib.sd_last_error(ctx.h)
    D = lib.sd_hog_feature_length(L, C.byref(p))
    A = torch.full((N, D), float("nan"), dtype=torch.float32, device="cuda")
    rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, C.byref(eyes), C.byref(p),
                          _capi.ptr(A), C.c_int64(D))
    assert rc == 0, lib.sd_last_error(ctx.h)
    rc = lib.sd_sync(ctx.h)
    assert rc == 0, lib.sd_last_error(ctx.h)
    return geo.cpu().numpy(), patches.cpu().numpy(), bins.cpu().numpy(), A.cpu().numpy()


def truth(oracle, frames, samples, cfg):
    """The oracle's geometry, patches, bins and feature rows of the samples."""
    variant, nc, cs, K = cfg
    fs = nc * cs
    op = oracle.HogParam(variant, nc, cs, K, 1.0)
    use_ref = oracle.ref_available()
    geo, pat, bins, feats = [], [], [], []
    for f, row in samples:
        img = frames[f]
        cx, cy, half = oracle.patch_geometry(row, op, [0], [1])
        ps = [oracle.resize_linear_u8(oracle.crop_patch_u8(img, int(cx[l]), int(cy[l]), int(half[l])), fs, fs) for l in range(L)]
        geo.append(np.stack([cx, cy, half], axis=1))
        pat.append(np.stack(ps))
        bins.append(np.stack([oracle.hog_orientation_bins(q.astype(np.float32), K) for q in ps]))
        feats.append(oracle.hog_transform(img, row, op, [0], [1], use_ref=use_ref))
    return np.stack(geo), np.stack(pat), np.stack(bins), np.stack(feats)


def compare(got, want, what):
    """Failure messages (empty when the kernel matches) and the worst feature error."""
    g_geo, g_pat, g_bins, g_A = got
    w_geo, w_pat, w_bins, w_A = want
    bad = []
    if not np.array_equal(g_geo, w_geo):
        bad.append(f"{what}: geometry differs in {int(np.sum(np.any(g_geo != w_geo, axis=2)))} windows")
    if not np.array_equal(g_pat, w_pat):
        bad.append(f"{what}: {int(np.sum(g_pat != w_pat))} resized patch pixels differ "
                   f"(in {int(np.sum(np.any(g_pat != w_pat, axis=(2, 3))))} windows)")
    if not np.array_equal(g_bins.astype(np.int32), w_bins):
        bad.append(f"{what}: {int(np.sum(g_bins.astype(np.int32) != w_bins))} orientation bins differ")
    if not np.array_equal(g_A[:, -1], w_A[:, -1]):
        bad.append(f"{what}: bias column differs")
    errs = [rel_err(g_A[i, :-1], w_A[i, :-1]) for i in range(len(w_A))]      # relative to the row's largest HOG feature
    worst = max(errs) if errs else 0.0
    if not worst <= FEATURE_TOL:
        bad.append(f"{what}: features {worst:.3g} from the reference (tolerance {FEATURE_TOL:g})")
    return bad, worst


# ---- host-only checks of the case lists --------------------------------------------------------------------------------
def test_configs_are_accepted_and_cover_every_kernel():
    for cfg in CONFIGS:
        assert accepted(cfg), (cfg, smem_layout(cfg))
    for v, nc, cs, K in LARGEST:                                # the next cell size no longer fits the shared memory
        assert not accepted((v, nc, cs + 1, K)) and smem_layout((v, nc, cs + 1, K))[1] > SMEM_LIMIT
    assert smem_layout((1, 1, 192, 4))[1] == 232064
    selectable = {(K, 5, cs) for K in (4, 9) for cs in (11, 10, 8, 6)} | {(4, 0, 0), (9, 0, 0), (0, 0, 0)}
    assert {kernel_of(c) for c in CONFIGS} == selectable
    assert {c[0] for c in CONFIGS} == {0, 1}


def route_plan(cfg):
    """[(layout kind, samples)] and the route counts of this configuration's windows over all layouts."""
    frames = _frames()
    common, small = route_samples(cfg)
    cap = smem_layout(cfg)[0]
    rois = []
    for f in (0, 1):                                            # the bounding box of the frame's windows, inside the frame
        wins = [(x, y, r) for s, r in common if s == f for x, y in _windows_of(r, int(r[1] - r[0]))]
        x0 = max(0, min(x for x, _, _ in wins)); y0 = max(0, min(y for _, y, _ in wins))
        x1 = min(W, max(x + int(r[1] - r[0]) for x, _, r in wins)); y1 = min(H, max(y + int(r[1] - r[0]) for _, y, r in wins))
        rois.append((x0, y0, x1 - x0, y1 - y0))
    plan, counts = [], Counter()
    for kind in LAYOUTS:
        lay = Layout(kind, frames, rois if kind == "roi" else None)
        samples = common + (small if kind == "frames" else [])
        for f, r in samples:
            P = int(r[1] - r[0])
            for x0, y0 in _windows_of(r, P):
                counts[route(cap, P, x0, y0, lay.desc[f])] += 1
        plan.append((lay, samples))
    return frames, plan, counts


def allowed_routes(cfg):
    return set(ROUTES) - (set() if smem_layout(cfg)[0] >= TMA_BOXES[0] ** 2 else {"tma"})


def _route_table(rows):
    lines = [f"{'config (variant, nc, cs, K)':<28}{'fs':>5}" + "".join(f"{r:>10}" for r in ROUTES)]
    for cfg, counts in rows:
        lines.append(f"{str(cfg):<28}{cfg[1] * cfg[2]:>5}" + "".join(f"{counts[r]:>10}" for r in ROUTES))
    return "\n".join(lines)


def test_route_cases_cover_every_route_each_layout_allows():
    rows = []
    for cfg in ROUTE_CONFIGS:
        _, _, counts = route_plan(cfg)
        rows.append((cfg, counts))
        assert {r for r in ROUTES if counts[r]} == allowed_routes(cfg), (cfg, counts)
    assert allowed_routes((1, 1, 4, 1)) == set(ROUTES) - {"tma"}
    print("\n" + _route_table(rows))


def test_sweep_resizes_are_pinned_by_cv2_goldens():
    """Every (P, fs) the configuration sweep resizes is a cv2 pair of resize_cv2_wide.npz (test_oracle.py pins the oracle's
    resize to them)."""
    g = np.load(os.path.join(GOLDEN, "resize_cv2_wide.npz"))
    for cfg in CONFIGS:
        fs = cfg[1] * cfg[2]
        for P in _wide.sweep_windows(fs):
            assert f"dst_{P}_{fs}" in g.files, (cfg, P)


def _hog_patch(rng, fs, k):
    """A seeded fs x fs patch: noise, blurred noise, or noise with a zero border band (as the zero padding of a window over a
    frame edge leaves, which gives K = 1 its gx = 0 pixels)."""
    img = rng.integers(0, 256, (fs, fs)).astype(np.float32)
    if k == 1:
        img = np.round((img + np.roll(img, 1, 0) + np.roll(img, 1, 1) + np.roll(img, (1, 1), (0, 1))) / 4)
    if k == 2:
        img[: max(1, fs // 3)] = 0
        img[:, : max(1, fs // 4)] = 0
    return img


def test_oracle_hog_core_matches_hog_c_at_every_config(oracle):
    """The oracle's restatement of hog.c (the truth of the GPU tests below when oracle/_ref is absent) against the
    reference's hog.c, bit for bit, at every sweep configuration and both variants."""
    if not oracle.ref_available():
        pytest.skip("oracle/_ref (the reference's hog.c) is not built")
    rng = np.random.default_rng(31)
    for _, nc, cs, K in CONFIGS:
        for variant in (0, 1):
            for k in range(3):
                img = _hog_patch(rng, nc * cs, k)
                a = oracle.hog_core(img, cs, K, variant)
                b = oracle.hog_core(img, cs, K, variant, use_ref=True)
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (variant, nc, cs, K, k)


# ---- GPU -------------------------------------------------------------------------------------------------------------------
def sweep_samples(fs):
    """One sample per window size of the sweep: eyes centred, landmark 2 over the top-left corner, landmark 3 inside."""
    return [_sample(k % 2, P, (-(P // 4), -(P // 4)), (53, 37)) for k, P in enumerate(_wide.sweep_windows(fs))]


@pytest.mark.gpu
def test_configuration_sweep(sd, oracle):
    """Every configuration of CONFIGS at windows below, equal to, twice and far above fs, in a batch the TMA route serves."""
    ctx = sd.default_context()
    frames = _frames()
    lay = Layout("tma", frames)
    ib, keep, _ = device_batch(lay)
    bad = []
    print(f"\nhog.c truth: {oracle.ref_available()}")
    for cfg in CONFIGS:
        fs = cfg[1] * cfg[2]
        samples = sweep_samples(fs)
        got = run_kernel(ctx, ib, samples, cfg)
        want = truth(oracle, frames, samples, cfg)
        for i, (_, r) in enumerate(samples):
            P = int(r[1] - r[0])
            b, worst = compare(tuple(a[i:i + 1] for a in got), tuple(a[i:i + 1] for a in want), f"{cfg} P={P}")
            bad += b
            print(f"{str(cfg):<18} fs={fs:<4} P={P:<4} worst feature error {worst:.2e}{'  FAIL' if b else ''}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_every_window_route(sd, oracle):
    """The route cases of ROUTE_CONFIGS in every layout: exact taps, features within tolerance of the reference, and the
    features of every window bit-identical across the layouts (so across the routes that serve it)."""
    ctx = sd.default_context()
    bad, rows = [], []
    for cfg in ROUTE_CONFIGS:
        frames, plan, counts = route_plan(cfg)
        rows.append((cfg, counts))
        want_all = None
        first = None
        for lay, samples in plan:
            ib, keep, miss = device_batch(lay)
            got = run_kernel(ctx, ib, samples, cfg)
            want = truth(oracle, frames, samples, cfg)
            b, worst = compare(got, want, f"{cfg} {lay.kind}")
            bad += b
            print(f"{str(cfg):<16} {lay.kind:<7} {len(samples):>3} samples  worst feature error {worst:.2e}{'  FAIL' if b else ''}")
            n = len(plan[0][1])                                 # the samples every layout shares come first
            if first is None:
                first = got[3][:n]
            elif not np.array_equal(got[3][:n].view(np.uint32), first.view(np.uint32)):
                rows_bad = np.flatnonzero(np.any(got[3][:n].view(np.uint32) != first.view(np.uint32), axis=1))
                bad.append(f"{cfg} {lay.kind}: features of samples {rows_bad.tolist()[:8]} differ from the tma layout's")
            if miss is not None and miss.cpu().numpy().any():
                bad.append(f"{cfg} roi: d_roi_miss set although the ROI covers every window")
        assert {r for r in ROUTES if counts[r]} == allowed_routes(cfg)
    print(_route_table(rows))
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
def test_roi_miss_is_flagged_per_frame(sd, oracle):
    """Windows that reach at least fs rows below the uploaded ROI (but stay in the frame) flag their frame, through the staged
    and the unstaged route; a frame whose ROI covers its windows is not flagged and matches the oracle."""
    cfg = (1, 5, 6, 4)
    fs = 30
    ctx = sd.default_context()
    frames = _frames()
    frames = [frames[0], frames[1], frames[0]]
    assert largest_staged(smem_layout(cfg)[0]) < 120
    # frame 0: a staged window of 80 rows from y = 100 (30 rows below the ROI); frame 1: an unstaged one of 120 rows (70);
    # frame 2: the same windows, with its whole frame uploaded
    samples = [_sample(0, 80, (60, 100), (200, 20), eyes=(100, 40)), _sample(1, 120, (60, 100), (200, 10), eyes=(100, 60)),
               _sample(2, 80, (60, 100), (200, 20), eyes=(100, 40)), _sample(2, 120, (60, 100), (200, 10), eyes=(100, 60))]
    lay = Layout("roi", frames, [(0, 0, W, 150), (0, 0, W, 150), (0, 0, W, H)])
    ib, keep, miss = device_batch(lay)
    got = run_kernel(ctx, ib, samples, cfg)
    assert miss.cpu().numpy().tolist() == [1, 1, 0]
    want = truth(oracle, frames, samples[2:], cfg)
    bad, worst = compare(tuple(a[2:] for a in got), want, "roi covering frame 2")
    print(f"roi miss: flags {miss.cpu().numpy().tolist()}, covered frame worst feature error {worst:.2e}")
    assert not bad, "\n".join(bad)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,message", [
    ((1, 5, 37, 4), "more than 227 KB"), ((1, 16, 10, 4), "more than 227 KB"), ((1, 1, 193, 4), "more than 227 KB"),
    ((1, 1, 3, 4), "4..256 px"), ((1, 1, 257, 4), "4..256 px")], ids=["5x37", "16x10", "1x193", "fs3", "fs257"])
def test_rejected_configurations_launch_nothing(sd, cfg, message):
    """Configurations outside the kernel's limits are SD_ERR_INVALID before any launch; the output keeps its sentinel."""
    import torch
    from superviseddescent_b200 import _capi
    lib = _capi.lib()
    ctx = sd.default_context()
    frames = _frames()
    ib, keep, _ = device_batch(Layout("tma", frames))
    assert smem_layout(cfg)[1] > SMEM_LIMIT or not 3 < cfg[1] * cfg[2] <= 256
    x = torch.from_numpy(np.stack([_sample(0, 40, (10, 10), (50, 50))[1]])).cuda()
    p, eyes = _param(cfg), _eyes()
    D = L * cfg[1] * cfg[1] * _dd(cfg[0], cfg[3]) + 1
    A = torch.full((1, D), 7.0, dtype=torch.float32, device="cuda")
    before = ctx.launches()
    rc = lib.sd_hog_batch(ctx.h, C.byref(ib), None, _capi.ptr(x), C.c_int64(2 * L), 1, L, C.byref(eyes), C.byref(p),
                          _capi.ptr(A), C.c_int64(D))
    assert rc == 1, (rc, lib.sd_last_error(ctx.h))
    assert message in lib.sd_last_error(ctx.h).decode()
    assert ctx.launches() == before
    assert lib.sd_sync(ctx.h) == 0
    assert bool(torch.all(A == 7.0))


@pytest.mark.gpu
def test_degenerate_sample_and_bad_image_index_flag_the_next_sync(sd):
    """An inter-eye distance whose half patch rounds to 0, and an image index outside the batch: the launch succeeds and the
    next sd_sync reports SD_ERR_INVALID with its message; the sync after that is clean."""
    import torch
    from superviseddescent_b200 import _capi
    lib = _capi.lib()
    ctx = sd.default_context()
    ib, keep, _ = device_batch(Layout("tma", _frames()))
    cfg = (1, 5, 6, 4)
    p, eyes = _param(cfg), _eyes()
    D = lib.sd_hog_feature_length(L, C.byref(p))
    A = torch.zeros((1, D), dtype=torch.float32, device="cuda")
    degenerate = np.array([[100, 100.5, 50, 60, 80, 80, 50, 60]], dtype=np.float32)        # IED 0.5: half = round(0.25) = 0
    good = _sample(0, 40, (10, 10), (50, 50))[1][None]
    for row, idx, message in ((degenerate, 0, "empty HOG patch"), (good, 2, "image index out of range")):
        x = torch.from_numpy(row).cuda()
        d_idx = torch.tensor([idx], dtype=torch.int32, device="cuda")
        rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(d_idx), _capi.ptr(x), C.c_int64(2 * L), 1, L, C.byref(eyes),
                              C.byref(p), _capi.ptr(A), C.c_int64(D))
        assert rc == 0, lib.sd_last_error(ctx.h)
        assert lib.sd_sync(ctx.h) == 1
        assert message in lib.sd_last_error(ctx.h).decode()
        assert lib.sd_sync(ctx.h) == 0
