"""The per-element HOG bars of tests/hog_ref64.py on the CPU: they accept, with margin, the reference's own hog.c (oracle/_ref),
the oracle's restatement orc_hog_core and the kernel-order float32 emulation, and they reject planted defects by more than 4x.
For each defect the old max-norm check (conftest.rel_err, the largest error over the largest reference value, held at 1e-4 and
1e-5 by the HOG GPU tests) is printed beside it, to show which defects that check lets through."""
import numpy as np
import pytest

import hog_ref64 as R
from conftest import rel_err

REJECT = 4.0
ACCEPT = 1.0                  # every bar is a bound that a single dominant rounding (a polar ho, the store) can nearly attain


def _u8(H, W, cs, seed):
    return R.blind_spot_frame(H, W, seed=seed, cs=cs)


def _float(C, H, W, cs, K, bil, seed, scale=1.0):
    base = np.stack([R.blind_spot_frame(H, W, seed=seed + c, cs=cs) for c in range(C)]).astype(np.float32)
    base += np.random.default_rng(seed).uniform(-0.3, 0.3, base.shape).astype(np.float32)
    side = min(3 * cs + 4, H // 3, W // 3)
    base[:, H - side:, W - side:] = 77.0
    return R.decided_float_frame((base * np.float32(scale)).astype(np.float32), K, bil, seed=seed, amp=0.25 * scale)


# (H, W, cs, K): every K of {1, 2, 4, 9, 16}, cell sizes 1 to 32
GREY = [(20, 30, 1, 2), (31, 29, 2, 9), (37, 53, 3, 16), (40, 48, 4, 4), (45, 50, 5, 1), (64, 64, 8, 16), (50, 45, 11, 4),
        (70, 70, 16, 9), (80, 75, 17, 2), (70, 70, 32, 9), (100, 90, 32, 16)]
# (channels, H, W, cs, K, bilinear, scale)
FLOAT = [(1, 40, 48, 4, 4, False, 1.0), (1, 36, 44, 4, 1, True, 1.0), (3, 40, 48, 4, 9, True, 1.0), (3, 40, 48, 8, 2, False, 1 / 255),
         (16, 33, 41, 3, 16, True, 1.0), (16, 30, 34, 1, 4, False, 1.0), (3, 70, 70, 32, 9, True, 1.0), (1, 61, 83, 6, 2, True, 1 / 255)]
# (H, W, cs, K)
POLAR = [(30, 37, 4, 4), (41, 29, 8, 9), (20, 20, 1, 1), (33, 35, 3, 16), (70, 66, 32, 2)]


def _ref(oracle):
    from oracle import vl_hog_polar_ref, vl_hog_ref
    vl_hog_ref.build()
    vl_hog_polar_ref.build()
    return oracle.ref_available() and vl_hog_ref.available() and vl_hog_polar_ref.available()


def _line(what, truth, bar, legs):
    parts = [f"{name} {R.worst(got, truth, bar):.3f}" for name, got in legs]
    return f"{what:<48} " + "  ".join(parts)


def test_bars_accept_hog_c_orc_and_the_kernel_order(oracle):
    """Every accepted arithmetic stays within its bar; the worst error / bar of each is printed."""
    from oracle import vl_hog_polar_ref, vl_hog_ref
    have_ref = _ref(oracle)
    worst = {}
    lines = []

    def check(what, truth, bar, legs):
        lines.append(_line(what, truth, bar, legs))
        for name, got in legs:
            r = R.worst(got, truth, bar)
            worst[name] = max(worst.get(name, 0.0), r)
            assert r <= ACCEPT, (what, name, r)

    for H, W, cs, K in GREY:
        img = _u8(H, W, cs, seed=H + cs)
        px = R.image_pixels(img, K)
        assert np.array_equal(px.bins[0], oracle.hog_orientation_bins(img.astype(np.float32), K))
        for v in (0, 1):
            t, b = R.truth(px, cs, K, v)
            legs = [("emulation", R.emulate(px, cs, K, v)), ("orc_hog_core", oracle.hog_core(img.astype(np.float32), cs, K, v))]
            if have_ref:
                legs.append(("hog.c", oracle.hog_core(img.astype(np.float32), cs, K, v, use_ref=True)))
            check(f"u8 {W}x{H} cs {cs} K {K} variant {v}", t, b, legs)
    for C, H, W, cs, K, bil, scale in FLOAT:
        f = _float(C, H, W, cs, K, bil, seed=C + H + cs, scale=scale)
        px = R.image_pixels(f if C > 1 else f[0], K, bil)
        for v in (0, 1):
            t, b = R.truth(px, cs, K, v)
            legs = [("emulation", R.emulate(px, cs, K, v))]
            if have_ref:
                legs.append(("hog.c", vl_hog_ref.vl_hog(f, cs, K, v, bil)))
            check(f"float x{scale:.3g} c {C} {W}x{H} cs {cs} K {K} bil {int(bil)} v {v}", t, b, legs)
    for H, W, cs, K in POLAR:
        for directed in (True, False):
            for bil in (False, True):
                m, a = R.polar_field(H, W, seed=H + K, K=K, directed=directed, bilinear=bil)
                px = R.polar_pixels(m, a, K, directed, bil)
                for v in (0, 1):
                    t, b = R.truth(px, cs, K, v)
                    legs = [("emulation", R.emulate(px, cs, K, v))]
                    if have_ref:
                        legs.append(("hog.c", vl_hog_polar_ref.vl_hog_polar(m, a, cs, K, v, directed, bil)))
                    check(f"polar {W}x{H} cs {cs} K {K} dir {int(directed)} bil {int(bil)} v {v}", t, b, legs)
    print("\n" + "\n".join(lines))
    print("worst error / bar: " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()) + ("" if have_ref else " (hog.c not built)"))


def _voting(px, where):
    """An interior voting pixel: 'centre' (texture), 'edge' (beside the strong step edge), 'border' (first interior row or
    column) or 'run4' (the fourth pixel of a 4-pixel gradient run of the landmark kernel, interior x = 4 mod 4 from 1)."""
    H, W = px.shape
    ok = (px.bins[0] >= 0) & (px.m > 0)
    yy, xx = np.nonzero(ok)
    if where == "centre":
        target = (H // 2, W // 2)
    elif where == "edge":
        target = (H // 5 + 1, max(2, W // 5) + 1)
    elif where == "border":
        target = (1, W // 2)
    else:
        sel = (xx - 1) % 4 == 3
        yy, xx = yy[sel], xx[sel]
        target = (H // 2, W // 2)
    i = np.argmin((yy - target[0]) ** 2 + (xx - target[1]) ** 2)
    return int(yy[i]), int(xx[i])


def _weak_pixel(px, cs, K):
    """The voting pixel nearest the centre of the cell whose largest feature is the smallest non-zero one in the frame: a
    low-contrast cell beside a strong edge, whose features sit far below the frame's largest."""
    t, _ = R.truth(px, cs, K, 1)
    top = np.max(t, axis=0)
    top = np.where(top > 0, top, np.inf)
    cy, cx = np.unravel_index(np.argmin(top), top.shape)
    ok = (px.bins[0] >= 0) & (px.m > 0)
    yy, xx = np.nonzero(ok)
    i = np.argmin((yy - (cy + 0.5) * cs) ** 2 + (xx - (cx + 0.5) * cs) ** 2)
    return int(yy[i]), int(xx[i])


def _edge_cell_pixel(px, cs, K):
    """A weak voting pixel (modulus <= 3) inside a cell that the strong edge crosses, voting into another bin than the edge's:
    its bin holds a feature far below the frame's largest, the blind spot of a max-norm check."""
    H, W = px.shape
    b = px.bins[0]
    strong = px.m >= 100
    best = None
    for cy in range(H // cs):
        for cx in range(W // cs):
            sl = (slice(cy * cs, (cy + 1) * cs), slice(cx * cs, (cx + 1) * cs))
            if not strong[sl].any():
                continue
            edge_bins = set(np.unique(b[sl][strong[sl]]))
            weak = (px.m[sl] > 0) & (px.m[sl] <= 3) & ~np.isin(b[sl], list(edge_bins)) & (b[sl] >= 0)
            yy, xx = np.nonzero(weak)
            if yy.size and (best is None or strong[sl].sum() > best[0]):
                best = (strong[sl].sum(), cy * cs + int(yy[0]), cx * cs + int(xx[0]))
    return best[1], best[2]


def _swap_pixel(px):
    """A bilinear pixel with two bins whose weights are far from equal (None at K = 1: one bin only)."""
    cand = np.argwhere((px.bins[1] >= 0) & (np.abs(px.wo32[1] - 0.5) > 0.2))
    return tuple(int(v) for v in cand[len(cand) // 2]) if len(cand) else None


def _defect_cases():
    """(name, px, cs, K, variant, defect, tile) for every planted defect, each on inputs where it is observable."""
    out = []
    for H, W, cs, K in [(40, 48, 4, 4), (64, 64, 8, 9), (70, 70, 16, 16)]:
        px = R.image_pixels(_u8(H, W, cs, seed=H + cs), K)
        tag = f"u8 cs {cs} K {K}"
        for where in ("centre", "edge", "border", "run4"):
            y, x = _voting(px, where)
            out.append((f"vote dropped ({where})", tag, px, cs, K, 1, ("drop", y, x), None))
        y, x = _weak_pixel(px, cs, K)
        out.append(("vote dropped (weak cell)", tag, px, cs, K, 1, ("drop", y, x), None))
        out.append(("vote into bin k + 1 (weak cell)", tag, px, cs, K, 1, ("bin", y, x, 1), None))
        y, x = _voting(px, "centre")
        out.append(("vote into bin k + 1", tag, px, cs, K, 1, ("bin", y, x, 1), None))
        out.append(("vote into bin k + K", tag, px, cs, K, 1, ("bin", y, x, K), None))
        out.append(("w1 / w2 swapped, column 1", tag, px, cs, K, 0, ("swap_w_column", 1), None))
        out.append(("w1 / w2 swapped, last column", tag, px, cs, K, 1, ("swap_w_column", W - 2), None))
        out.append(("edge block factor unclamped", tag, px, cs, K, 0, ("edge_factor",), None))
        for q in ("haf", "hbf", "hcf"):
            out.append((f"no 0.2 clamp on {q}", tag, px, cs, K, 1, ("no_clamp", q), None))
        out.append(("texture dim of three factors", tag, px, cs, K, 1, ("texture3",), None))
        T = max(1, min(14, 110 // cs - 4))
        if R.grid(W, H, cs)[0] > T:
            out.append(("dense halo column unvoted", tag, px, cs, K, 1, ("halo_unvoted",), T))
    # the blind spot of the max-norm check: a weak vote beside a strong edge, in a cell dominated by it
    for H, W, cs, K in [(64, 64, 8, 9), (70, 70, 16, 16), (100, 90, 32, 16)]:
        px = R.image_pixels(_u8(H, W, cs, seed=H + cs), K)
        y, x = _edge_cell_pixel(px, cs, K)
        for v in (0, 1):
            tag = f"u8 cs {cs} K {K} variant {v}"
            out.append(("vote dropped (beside the edge)", tag, px, cs, K, v, ("drop", y, x), None))
            out.append(("vote into bin k + 1 (beside the edge)", tag, px, cs, K, v, ("bin", y, x, 1), None))
    # every bilinear image case of the GPU tests, float and 8-bit: drop, bin k + 1 and w0 / w1 exchanged
    for case in R.IMAGE_CASES:
        C, layout, cs, K, H, W, scale = case
        for kind in ("f32", "u8"):
            f = R.image_case_frame(case, kind, True)
            px = R.image_pixels(f if C > 1 else f[0], K, True, check_margin=kind == "f32")
            tag = f"{kind} c {C} cs {cs} K {K} bilinear"
            y, x = _voting(px, "centre")
            out.append(("bilinear vote dropped", tag, px, cs, K, 1, ("drop", y, x), None))
            out.append(("bilinear vote into bin k + 1", tag, px, cs, K, 1, ("bin", y, x, 1), None))
            p = _swap_pixel(px)
            if p is not None:
                out.append(("bilinear w0 / w1 exchanged", tag, px, cs, K, 1, ("swap_wo",) + p, None))
    for cs, K in [(4, 4), (8, 9)]:
        m, a = R.polar_field(30, 37, seed=cs, K=K, directed=True, bilinear=False)
        m = (np.abs(m) * np.float32(1e-6)).astype(np.float32)              # low contrast everywhere: small energies
        px = R.polar_pixels(m, a, K, True, False)
        out.append(("1e-4 of the block factor missing", f"polar 1e-6 cs {cs} K {K}", px, cs, K, 1, ("no_eps",), None))
    return out


def test_bars_reject_planted_defects():
    """Each planted defect exceeds its bar by more than 4x; the old max-norm check's value is printed beside it."""
    lines, bad, through = [], [], set()
    for name, tag, px, cs, K, v, defect, tile in _defect_cases():
        t, b = R.truth(px, cs, K, v)
        got = R.emulate(px, cs, K, v, defect, tile)
        r = R.worst(got, t, b)
        with np.errstate(invalid="ignore"):
            old = rel_err(got, t)
        lines.append(f"{name:<34} {tag:<22} error / bar {r:10.3g}   rel_err {old:.2e}"
                     f"{'  (passes 1e-5)' if old <= 1e-5 else '  (passes 1e-4)' if old <= 1e-4 else ''}")
        if old <= 1e-4:
            through.add(name)
        if not r > REJECT:
            bad.append(f"{name} {tag}: {r:.3g}")
    print("\n" + "\n".join(lines))
    print("let through by the max-norm checks somewhere: " + (", ".join(sorted(through)) or "none"))
    assert not bad, bad


def test_bars_of_a_flat_frame_are_zero():
    """A frame without gradients has all-zero truth and bars, so every feature must be exactly 0."""
    img = np.full((24, 28), 93, np.uint8)
    for v in (0, 1):
        t, b = R.truth(R.image_pixels(img, 4), 4, 4, v)
        assert not t.any() and not b.any()
        assert R.worst(np.full(t.shape, 1e-30, np.float32), t, b) == np.inf
