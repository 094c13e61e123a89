"""The landmark HOG projection in two kernels: hog_patch_kernel leaves each patch's cell histograms in the first 2K cells
floats of its feature slice and hog_normalise_kernel (csrc/sd_hog.cu) normalises them in place, several patches per CTA.

Against the reference's hog.c (through the oracle, as tests/test_gpu_hog_configs.py) at both variants, K = 1 and K = 16,
run-time configurations with more than 32 cells (up to 289, more than one CTA's threads), batches whose patch count is not
a multiple of the normalisation kernel's patches per CTA, on the TMA and the byte-loop staging routes; and with an odd row
stride ld, so that the slices start at every float offset: the same rows bit for bit, the floats past the feature row
untouched.
"""
import ctypes as C

import numpy as np
import pytest

import test_gpu_hog_configs as hc

L = hc.L
# (variant, num_cells, cell_size, num_bins): compiled-in schedules, K = 1 and 16, 36 / 64 / 144 / 256 / 289 cells
CONFIGS = [(1, 5, 11, 4), (0, 5, 10, 9), (1, 1, 4, 1), (0, 4, 3, 1), (1, 6, 7, 5), (1, 8, 8, 16), (0, 12, 6, 16),
           (1, 16, 9, 4), (0, 17, 2, 4)]
N = 7


def per_cta(cfg):
    """hog_normalise_kernel's patches per CTA (launch_hog): one thread per cell of 256."""
    cells = cfg[1] * cfg[1]
    return 256 // cells if cells < 256 else 1


def _samples(fs):
    """N samples on frames 0 and 1, windows from about fs to 2 fs, one landmark over the top-left corner."""
    out = []
    for k in range(N):
        P = 2 * ((fs + k * fs // 6) // 2) + 2
        out.append(hc._sample(k % 2, P, (-(P // 4), -(P // 3)), (53 + 7 * k, 37 + 5 * k)))
    return out


def _features(ctx, ib, samples, cfg, ld):
    """sd_hog_batch into an (N, ld) buffer prefilled with a sentinel."""
    import torch
    from superviseddescent_b200 import _capi
    lib = _capi.lib()
    x = torch.from_numpy(np.stack([r for _, r in samples])).cuda()
    idx = torch.tensor([f for f, _ in samples], dtype=torch.int32, device="cuda")
    p, eyes = hc._param(cfg), hc._eyes()
    A = torch.full((len(samples), ld), -3.0, dtype=torch.float32, device="cuda")
    rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), len(samples), L, C.byref(eyes),
                          C.byref(p), _capi.ptr(A), C.c_int64(ld))
    assert rc == 0, lib.sd_last_error(ctx.h)
    assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
    return A.cpu().numpy()


def test_cases_cover_the_split():
    assert {c[0] for c in CONFIGS} == {0, 1} and {1, 16} <= {c[3] for c in CONFIGS}
    assert max(c[1] * c[1] for c in CONFIGS) > 256
    assert any((N * L) % per_cta(c) for c in CONFIGS)
    for c in CONFIGS:
        assert hc.accepted(c), c
        D = L * c[1] * c[1] * hc._dd(c[0], c[3]) + 1
        assert 2 * c[3] * c[1] * c[1] * L < D                     # the histograms fit the slices they are written to


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["tma", "bytes"])
def test_split_matches_hog_c_at_any_row_stride(sd, oracle, kind):
    ctx = sd.default_context()
    frames = hc._frames()
    lay = hc.Layout(kind, frames)
    ib, keep, _ = hc.device_batch(lay)
    bad = []
    for cfg in CONFIGS:
        samples = _samples(cfg[1] * cfg[2])
        got = hc.run_kernel(ctx, ib, samples, cfg)
        want = hc.truth(oracle, frames, samples, cfg)
        b, worst = hc.compare(got, want, f"{cfg} {kind}")
        bad += b
        D = got[3].shape[1]
        ld = D + 2 if D % 2 else D + 1                               # odd: row r's slices start at r mod 4 floats
        A = _features(ctx, ib, samples, cfg, ld)
        if not np.array_equal(A[:, :D].view(np.uint32), got[3].view(np.uint32)):
            bad.append(f"{cfg} {kind}: rows at ld = {ld} differ from those at ld = D = {D}")
        if not np.all(A[:, D:] == -3.0):
            bad.append(f"{cfg} {kind}: floats past the feature row were written")
        print(f"{str(cfg):<16} {kind:<6} patches {N * L} per CTA {per_cta(cfg)} worst feature error {worst:.2e}"
              f"{'  FAIL' if b else ''}")
    assert not bad, "\n".join(bad)
