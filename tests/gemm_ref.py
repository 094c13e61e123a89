"""Float64 references and per-element error bars for the Gram, predict and cascade-update kernels, plus a numpy restatement of
the tensor-core Gram arithmetic (sd_gram_tc.cu) that the bars are checked against without a GPU.

Every bar is per element, so an error in a small entry cannot hide behind the largest one:
    Gram        |G_ij - G^_ij| <= tau(mode, N) * ||a_i|| * ||a_j||        (a_j = column j of [A | B])
    predict     |Y_ij - Y^_ij| <= TAU_PREDICT * sum_k |a_ik x_kj|
By Cauchy-Schwarz sum_k |a_ik a_jk| <= ||a_i|| ||a_j||, so anything bounded relative to the sum of the absolute products of an
entry is bounded relative to the product of the column norms.

tau of the Gram (u = 2^-24, the unit roundoff of fp32 round-to-nearest; rounding errors of long sums are modelled as a random
walk, lambda * sqrt(R) * u for R roundings, lambda = 8, the probabilistic bound of Higham & Mary, SISC 2019):
  mode 0 (3xTF32, truncated hi): hi is the raw value with the low 13 bits ignored, so |lo| < 2^-10 |a|; the dropped lo*lo term is
      below 2^-20 |a_i a_j|, and lo = rna_tf32(a - hi) is off by at most 2^-11 |lo| <= 2^-21 |a|, which enters twice (hi*lo, lo*hi):
      split error <= 2^-20 + 2 * 2^-21 = 2^-19 per product.  Sums: 3 x 16 accumulating k8 MMAs per 128-sample chunk, then one
      fp32 add per chunk into the running sum: R = 48 + ceil(N / 128).
  mode 3 (3xTF32, rounded hi): |lo| <= 2^-11 |a|: lo*lo <= 2^-22, lo rounding 2 * 2^-22: split error <= 3 * 2^-22.  Same sums.
  mode 1 (single TF32 pass): each operand loses up to 2^-10 of itself: split error <= 2 * 2^-10 + 2^-20 < 2^-8.7; one MMA per k8
      step: R = 16 + ceil(N / 128).
  mode 2 (fp32 SIMT): exact operands, one fp32 FMA chain per contraction range (at most N long, the split-K reduce adds at most
      64 partials): R = N + 64.
"""
import math

import numpy as np

U = 2.0 ** -24
LAMBDA = 8.0
KC = 128                                    # samples per accumulation chunk of the tensor-core kernel

SPLIT = {0: 2.0 ** -19, 3: 3 * 2.0 ** -22, 1: 2 * 2.0 ** -10 + 2.0 ** -20, 2: 0.0}
MMA_STEPS = {0: 48, 3: 48, 1: 16}


def tau_gram(mode: int, n: int) -> float:
    """Per-element bar of the Gram relative to ||a_i|| ||a_j|| for gram mode `mode` and n samples (module docstring)."""
    chunks = -(-n // KC)
    rounds = n + 64 if mode == 2 else MMA_STEPS[mode] + chunks
    return SPLIT[mode] + LAMBDA * math.sqrt(rounds) * U


# predict: predict_rows_kernel sums 32 fp32 FMAs per chunk (gemm_nn_kernel 16), the chunk sums in double, then one rounding to
# fp32: |err| <= (gamma_32 + u) sum_k |a_ik x_kj| with gamma_32 ~ 32 u (deterministic worst case: 33 u = 2.0e-6)
TAU_PREDICT = 33 * U


def gram_ref(A, B=None):
    """[A^T A | A^T B] in float64 from the float32 inputs."""
    S = np.asarray(A, np.float64) if B is None else np.hstack([np.asarray(A, np.float64), np.asarray(B, np.float64)])
    A64 = np.asarray(A, np.float64)
    return A64.T @ S


def gram_bar(A, B, mode: int):
    """tau(mode, N) * ||a_i|| * ||a_j|| for i < D, j < D + M."""
    A64 = np.asarray(A, np.float64)
    na = np.linalg.norm(A64, axis=0)
    nb = na if B is None else np.concatenate([na, np.linalg.norm(np.asarray(B, np.float64), axis=0)])
    return tau_gram(mode, A64.shape[0]) * np.outer(na, nb)


def gram_excess(G, A, B, mode: int):
    """max over the upper triangle of AtA and all of AtB of |G - G^| / bar (<= 1 passes), and the float64 reference.
    Only those entries are an output of sd_gram."""
    D = np.asarray(A).shape[1]
    ref = gram_ref(A, B)
    bar = gram_bar(A, B, mode)
    ratio = np.abs(np.asarray(G, np.float64)[:, :ref.shape[1]] - ref) / np.maximum(bar, 1e-300)
    ratio[:, :D][np.tril_indices(D, -1)] = 0.0
    return float(np.max(ratio)), ref


def predict_ref(A, X):
    A64, X64 = np.asarray(A, np.float64), np.asarray(X, np.float64)
    return A64 @ X64, TAU_PREDICT * (np.abs(A64) @ np.abs(X64))


# ---- numpy restatement of the tensor-core arithmetic (3xTF32, mode 0 / 3) ----
def trunc_tf32(x):
    """the operand as the tensor core sees it: low 13 mantissa bits ignored"""
    return (np.asarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def rna_tf32(x):
    """round to 10 mantissa bits, ties away from zero (cvt.rna.tf32.f32 on finite values)"""
    b = np.asarray(x, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def emulate_gram(A, B=None, unbiased=False, drop_lohi=False):
    """[A^T A | A^T B] as syrk_wgmma_kernel computes it: hi / lo split of both operands, the products lo*hi, hi*lo, hi*hi of every
    sample accumulated in fp32 inside each 128-sample chunk (a fresh accumulator per chunk), chunks folded into an fp32 running sum.
    Products of TF32 values are exact in fp32.  drop_lohi leaves out the lo*hi product (a defect the bars must catch)."""
    A = np.asarray(A, np.float32)
    S = A if B is None else np.hstack([A, np.asarray(B, np.float32)])
    N, D = A.shape
    hi_s = rna_tf32(S) if unbiased else trunc_tf32(S)
    lo_s = rna_tf32(S - hi_s)
    hi_a, lo_a = hi_s[:, :D], lo_s[:, :D]
    run = np.zeros((D, S.shape[1]), np.float32)
    for c0 in range(0, N, KC):
        sl = slice(c0, min(N, c0 + KC))
        terms = [] if drop_lohi else [lo_a[sl, :, None] * hi_s[sl, None, :]]
        terms += [hi_a[sl, :, None] * lo_s[sl, None, :], hi_a[sl, :, None] * hi_s[sl, None, :]]
        seq = np.stack(terms, axis=1).reshape(-1, D, S.shape[1])          # sample by sample, lo*hi, hi*lo, hi*hi
        acc = np.cumsum(seq, axis=0, dtype=np.float32)[-1]
        run = (run + acc).astype(np.float32)
    return run
