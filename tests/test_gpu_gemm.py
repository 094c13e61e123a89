"""sd_gram, sd_predict and sd_cascade_update against float64 at the edges of their tilings, with the per-element error bars of
gemm_ref.py: sample counts around the tensor-core threshold, the 16-sample stage and the 128-sample chunk; more upper tiles than
CTAs; long contractions; A and B apart or in one buffer; padded, odd and misaligned leading dimensions; every gram mode; every
route of the predict GEMM."""
import ctypes as C

import numpy as np
import pytest

import gemm_ref as R

pytestmark = pytest.mark.gpu
SENTINEL = np.float32(-12345.5)


def _features(rng, n, d):
    """HOG-like: non-negative, bounded by 0.4, correlated columns, bias column of ones"""
    base = rng.random((n, 8), dtype=np.float32)
    A = np.clip(0.05 * (base @ rng.random((8, d), dtype=np.float32)) + 0.1 * rng.random((n, d), dtype=np.float32), 0, 0.4)
    A = A.astype(np.float32)
    A[:, -1] = 1.0
    return A


def _padded(M, ld, guard_rows=3):
    """M in the first columns of a buffer with row pitch ld; pad columns and guard_rows extra rows hold NaN"""
    buf = np.full((M.shape[0] + guard_rows, ld), np.nan, np.float32)
    buf[:M.shape[0], :M.shape[1]] = M
    return buf


def _round4(x):
    return (x + 3) // 4 * 4


# (n, d, m, mode, layout, lda, ldg, shift)
#   layout "apart": A and B in separate NaN-padded buffers; "inplace": B is columns [d, d + m) of A's buffer (d_B = d_A + d)
#   lda / ldg: None = tight; ldg "odd" = d + m + 1 (scalar stores), "pad" = round4(d + m) + 8; shift: G base moved by that many floats
GRAM_CASES = [
    *[(n, 300, 8, 0, "apart", None, None, 0) for n in (1, 15, 63, 64, 65, 127, 128, 129, 3001)],
    (1000, 2300, 136, 0, "apart", None, None, 0),         # 18 x 20 tile grid: more upper tiles than CTAs
    (700, 4000, 44, 0, "inplace", 4048, "pad", 0),        # 528 upper tiles, 4 per CTA
    (333, 1001, 2, 0, "apart", None, "odd", 0),           # D + M = 1003
    (200_003, 300, 8, 0, "apart", None, None, 0),          # ~1560 chunks folded per element
    (200_003, 300, 8, 3, "apart", None, None, 0),
    (1500, 700, 44, 0, "inplace", 756, "pad", 1),         # NaN pad columns, G misaligned by one float
    (1500, 700, 44, 0, "inplace", 747, None, 0),          # lda % 4 != 0: the SIMT route
    (1500, 700, 44, 0, "apart", 705, "odd", 0),
    (777, 513, 3, 0, "apart", None, "pad", 1),
    (1500, 700, 44, 3, "inplace", 744, "odd", 0),
    (1500, 700, 44, 1, "apart", None, "pad", 1),
    (3001, 700, 44, 1, "apart", None, None, 0),
    (1500, 700, 44, 2, "apart", None, "odd", 0),
    (5000, 700, 44, 2, "apart", None, None, 0),           # 132 SIMT tiles, K > 2048: split-K + reduce
    (129, 300, 8, 2, "inplace", 309, None, 1),
]


def _gram_id(c):
    n, d, m, mode, layout, lda, ldg, shift = c
    return f"n{n}-d{d}-m{m}-mode{mode}-{layout}-lda{lda or 'tight'}-ldg{ldg or 'tight'}-shift{shift}"


@pytest.mark.parametrize("case", GRAM_CASES, ids=_gram_id)
def test_gram_vs_float64(sd, case):
    import torch
    from superviseddescent_b200 import _capi
    n, d, m, mode, layout, lda, ldg, shift = case
    rng = np.random.default_rng(n * 31 + d + m)
    A = _features(rng, n, d)
    B = (0.05 * rng.standard_normal((n, m))).astype(np.float32)
    ctx = sd.default_context()
    if layout == "inplace":
        lda = lda or d + m
        bufA = _padded(np.hstack([A, B]), lda)
        dA = torch.from_numpy(bufA).cuda()
        pB, ldb = _capi.ptr(dA.data_ptr() + 4 * d), lda
    else:
        lda = lda or d
        dA = torch.from_numpy(_padded(A, lda)).cuda()
        ldb = m + 3
        dB = torch.from_numpy(_padded(B, ldb)).cuda()
        pB = _capi.ptr(dB)
    w = d + m
    ldg = {None: w, "odd": w + 1, "pad": _round4(w) + 8}[ldg]
    guard = 4 * ldg
    flat = torch.full((shift + d * ldg + guard,), float(SENTINEL), dtype=torch.float32, device="cuda")
    ctx.set_gram_mode(mode)
    try:
        rc = _capi.lib().sd_gram(ctx.h, _capi.ptr(dA), C.c_int64(lda), pB, C.c_int64(ldb), n, d, m,
                                 _capi.ptr(flat.data_ptr() + 4 * shift), C.c_int64(ldg))
        assert rc == 0, _capi.lib().sd_last_error(ctx.h)
        torch.cuda.synchronize()
    finally:
        ctx.set_gram_mode(0)
    h = flat.cpu().numpy()
    G = h[shift:shift + d * ldg].reshape(d, ldg)
    assert np.all(h[:shift] == SENTINEL) and np.all(h[shift + d * ldg:] == SENTINEL), "write outside G"
    assert np.all(G[:, w:] == SENTINEL), "write into the pad columns of G"
    out = np.concatenate([G[:, :d][np.triu_indices(d)], G[:, d:w].ravel()])
    assert np.all(np.isfinite(out))
    excess, ref = R.gram_excess(G[:, :w], A, B, mode)
    rel = np.max(np.abs(G[:, :w] - ref)[np.triu(np.ones((d, w), bool))]) / np.max(np.abs(ref))
    print(f"{_gram_id(case)}: tau {R.tau_gram(mode, n):.2e}, max error / bar {excess:.3f}, max error / max|G| {rel:.2e}")
    assert excess <= 1.0


def _predict(sd, A_buf, lda, n, d, X, m):
    import torch
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    out = torch.full((max(n, 1), m + 1), float(SENTINEL), dtype=torch.float32, device="cuda")
    rc = _capi.lib().sd_predict(ctx.h, _capi.ptr(A_buf), C.c_int64(lda), n, d, _capi.ptr(X), m, _capi.ptr(out), C.c_int64(m + 1))
    assert rc == 0, _capi.lib().sd_last_error(ctx.h)
    Y = out.cpu().numpy()
    assert np.all(Y[:, m] == SENTINEL)
    return Y[:n, :m]


# (d, lda, rows, cols): D >= 1024 with lda % 4 == 0 and M <= 192 is the predict_rows route (256 rows per CTA, column groups of
# 48); the rest goes to gemm_nn, split over D when few output tiles exist (D >= 1024)
PREDICT_CASES = [
    (1024, 1024, (1, 255, 256, 257, 2000), (2, 44, 48, 49, 136, 192)),
    (17051, 17052, (1, 255, 256, 257, 2000), (2, 44, 48, 49, 136, 192)),
    (700, 700, (1, 257, 2000), (44, 200)),                   # gemm_nn, no split
    (2000, 2000, (257, 2000), (200,)),                       # gemm_nn split over D
    (1025, 1025, (1, 257, 2000), (44,)),                     # lda % 4 != 0: gemm_nn split over D
]


@pytest.mark.parametrize("d,lda,rows,cols", PREDICT_CASES, ids=lambda v: str(v) if np.isscalar(v) else None)
def test_predict_vs_float64(sd, d, lda, rows, cols):
    import torch
    rng = np.random.default_rng(d)
    A = (rng.standard_normal((max(rows), d)) * 0.1).astype(np.float32)
    dA = torch.from_numpy(_padded(A, lda)).cuda()
    Xall = (rng.standard_normal((d, max(cols))) * 0.02).astype(np.float32)
    ref_all, bar_all = R.predict_ref(A, Xall)          # the columns of a product are independent: slices serve every M
    worst = 0.0
    for m in cols:
        dX = torch.from_numpy(np.ascontiguousarray(Xall[:, :m])).cuda()
        for n in rows:
            Y = _predict(sd, dA, lda, n, d, dX, m)
            e = float(np.max(np.abs(Y - ref_all[:n, :m]) / bar_all[:n, :m]))
            worst = max(worst, e)
            assert e <= 1.0, f"D={d} lda={lda} N={n} M={m}: error / bar {e:.3f}"
    print(f"D={d} lda={lda}: max error / bar {worst:.3f}")


def _ied(x, right, left):
    """inter-eye distance as sd_device_ied evaluates it (float eye centres, double norm)"""
    L = x.shape[1] // 2
    f = np.float32
    rx, ry, lx, ly = (np.zeros(x.shape[0], f) for _ in range(4))
    for i in right:
        rx, ry = rx + x[:, i], ry + x[:, i + L]
    for i in left:
        lx, ly = lx + x[:, i], ly + x[:, i + L]
    ir, il = f(1) / f(len(right)), f(1) / f(len(left))
    dx = ((rx * ir) - (lx * il)).astype(np.float64)
    dy = ((ry * ir) - (ly * il)).astype(np.float64)
    return np.sqrt(dx * dx + dy * dy)


@pytest.mark.parametrize("d,lda,n", [(17051, 17052, 300), (1025, 1025, 300), (700, 700, 300)],
                         ids=["predict_rows", "gemm_nn_split", "gemm_nn"])
def test_cascade_update_with_ied_vs_float64(sd, d, lda, n):
    """x_next = x - (A X) (.) (1 / (1 / ied)) with inter-eye-distance normalisation (sd_cascade_update), on each GEMM route"""
    import torch
    from superviseddescent_b200 import _capi
    L = 68
    rng = np.random.default_rng(d + n)
    A = (rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    X = (rng.standard_normal((d, 2 * L)) * 0.02).astype(np.float32)
    x = (rng.random((n, 2 * L)) * 100 + 50).astype(np.float32)
    right, left = [36, 39], [42, 45]
    norm = _capi.NormalisationC(1, 2, 2, (C.c_int32 * 4)(*right, 0, 0), (C.c_int32 * 4)(*left, 0, 0))
    dA, dX, dx = torch.from_numpy(_padded(A, lda)).cuda(), torch.from_numpy(X).cuda(), torch.from_numpy(x).cuda()
    dxn = torch.full_like(dx, float(SENTINEL))
    ctx = sd.default_context()
    rc = _capi.lib().sd_cascade_update(ctx.h, _capi.ptr(dA), C.c_int64(lda), n, d, _capi.ptr(dX), 2 * L, _capi.ptr(dx),
                                       C.byref(norm), _capi.ptr(dxn))
    assert rc == 0, _capi.lib().sd_last_error(ctx.h)
    got = dxn.cpu().numpy().astype(np.float64)
    ied = _ied(x, right, left)
    inv_n = (np.float32(1) / (1.0 / ied).astype(np.float32)).astype(np.float64)      # 1 / normalisation, in float
    prod, pbar = R.predict_ref(A, X)
    upd = prod * inv_n[:, None]
    ref = x.astype(np.float64) - upd
    bar = pbar * inv_n[:, None] + 2 * R.U * (np.abs(upd) + np.abs(ref))
    e = float(np.max(np.abs(got - ref) / bar))
    print(f"cascade update D={d} lda={lda}: max error / bar {e:.3f}")
    assert e <= 1.0
