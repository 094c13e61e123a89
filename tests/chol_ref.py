"""Float64 truth, per-element error bars and numpy restatements for the solve behind sd_solve_gram and the learn path
(csrc/sd_linalg.cu): the regulariser, the bias-first elimination, the blocked Cholesky `cholesky_solve`, and the small
partial-pivot LU `lu_small_kernel`.

The system.  For D > 256 the kernels regularise G (the float32 upper triangle of [A^T A | A^T B], lambda added to the diagonal
in float32, not to the bias row unless regularise_last_row), eliminate the bias (last) row first with pivot p = G_bb and
s = G[:D-1, D-1], and factor what is left,
    S = G_ww + Lambda - s s^T / p,      S w = b = R_w - s r_b^T / p,      x_b = (r_b - s^T w) / p.
`Truth` solves that system in float64 from the float32 matrix the GPU receives.

The bar on w (Skeel-type, per element).  A backward perturbation |dS_jk| <= tau (|U^T||U|)_jk, |db_j| <= tau |b_j| (U: the
float64 Cholesky factor of S) moves w by dw = S^-1 (db - dS w).  Summed with absolute values this is Skeel's
|S^-1| (|U^T||U| |w| + |b|); the perturbations of different entries come from different rounding chains and have independent
signs, so through S^-1 they add as a random walk instead, and the bar is
    |w^ - w|_i <= lambda_rw * sqrt( sum_j (S^-1)_ij^2 * tau^2 * ( sum_k (|U^T||U|)_jk^2 w_k^2 + b_j^2 ) ),
lambda_rw = 8 (the probabilistic factor of Higham & Mary, SISC 2019, as in gemm_ref.py).  tau bounds one entry's backward error
(u = 2^-24; R roundings along the chain that produces the entry count sqrt(R) u, the random-walk model):
  - every entry of S and b is rounded once by the bias downdate (double, then float32) and once when lambda is added: 2 roundings;
  - an entry receives one trailing update per earlier 256-row panel, each a length-256 contraction added onto it: on the tensor
    cores 3 x 32 accumulating k8 MMAs in two 128-deep chunks plus the fold and the add (about 100 roundings), on the SIMT route
    one FMA per product (257 roundings, the larger, counted); ceil((D-1) / 256) panels;
  - inside its diagonal block: 4 sub-steps of 32 right-looking rank-1 FMAs and the panel GEMMs between them (128), the
    off-diagonal blocks of W = U_jj^-1 built from the 32 x 32 inverses by two chained products (2 x 128), the panel solve
    U_jj^-T P as a 128-deep GEMM with W^T and, on the second block row of a panel, the fused A^T P (2 x 128), one spare (128);
  - the back substitution: X_j = W Y_j (128) and one 128-deep update of Y per later block (128 per block).
  So R(D) = 2 + 257 * panels + 6 * 128 + 128 * (blocks + 1), about 3.5 D: the gamma_{3n+1} of Higham's Theorem 10.4 for the
  Cholesky solve, plus the explicit-inverse terms.
  - the trailing updates' operand split: an unbiased 3xTF32 product is off by at most SPLIT[3] = 3 * 2^-22 of |p_ki p_kj|, so
    it adds at most SPLIT[3] (|U^T||U|)_jk to an entry (gemm_ref.SPLIT).  Gram modes 0 and 3 both run the updates with the
    rounded hi part; mode 2 is exact operands (0); mode 1 is one TF32 pass, SPLIT[1] ~ 2^-9.
  tau(mode, D) = SPLIT_UPDATE[mode] + sqrt(R(D)) * u.
The bias row follows from w: |dx_b| <= |s|^T |dw| / p, plus its own rounding.

The learn path adds the Gram's own per-entry error E = (SPLIT + sqrt(R) u) ||a_i|| ||a_j|| (gemm_ref's split and rounding counts
of the centred columns, gram mode 0 or the SIMT route, whichever is larger; gemm_ref.gram_bar without its random-walk factor),
carried through S = G_ww - s s^T / p and b = R_w - s r_b / p to first order (E_S, E_b), inside the same random walk, so that
lambda_rw is applied once:  sum_j (S^-1)_ij^2 (sum_k E_S,jk^2 w_k^2 + E_b,j^2).

Gram mode 1 gets no bar on w: its single TF32 pass perturbs S by up to SPLIT[1] |U^T||U|, and when that reaches S's smallest
eigenvalue (Truth.split_can_break) the factorisation may find the matrix not positive definite and must then say so.

The normwise backward error eta = ||r|| / (||S|| ||x|| + ||b||) per right-hand side is compared with LAPACK float32 spotrs on the
same float32 S.  A backward perturbation tau' |U^T||U| raises eta by tau' * rho, rho = || |U^T||U| ||_F / ||S||_F, so the GPU may
exceed spotrs by the split term SPLIT_UPDATE[mode] * rho plus one rounding of x to float32 (u).

`cholesky_restated` restates cholesky_solve in numpy float32 (256-row panels of two 128-blocks, explicit W = U_jj^-1 and W^T,
the fused A^T P term, head and tail updates with the split emulated through gemm_ref.rna_tf32, back substitution with W); it
stands in for the kernels when the bars are checked without a GPU, and its `defect` argument plants the defects the bars must
reject.  `lu_restated` is lu_small_kernel operation by operation.
"""
import math

import numpy as np
import scipy.linalg as sl

import gemm_ref as R

U = R.U
LAMBDA_RW = R.LAMBDA
PB = 128                                    # Cholesky block
PANEL = 256                                 # factorisation panel: two blocks
LU_MAX_DIM = 256
SPLIT_UPDATE = {0: R.SPLIT[3], 3: R.SPLIT[3], 2: 0.0, 1: R.SPLIT[1]}
f32 = np.float32


def roundings(D: int) -> int:
    """R(D) of the module docstring for the (D - 1)-dimensional system left after the bias elimination"""
    n = D - 1
    panels, blocks = -(-n // PANEL), -(-n // PB)
    return 2 + 257 * panels + 6 * 128 + 128 * (blocks + 1)


def tau_entry(mode: int, D: int) -> float:
    """bound on the backward error of one entry of S or b, relative to (|U^T||U|)_jk or |b_j|"""
    return SPLIT_UPDATE[mode] + math.sqrt(roundings(D)) * U


# ---- the system the kernels solve ---------------------------------------------------------------------------------------
def sym_from_upper(G):
    """the full symmetric float64 matrix of the upper triangle of G's D x D part"""
    D = G.shape[0]
    T = np.triu(np.asarray(G[:, :D], np.float64))
    return T + np.triu(T, 1).T


def lambda_matrix_norm(G, param: float, n_train: int) -> float:
    """lambda_kernel: param * (float)||sym(G)||_F / (float)n in float32, from the float64 norm of the float32 matrix"""
    s = math.sqrt(float(np.sum(sym_from_upper(G) ** 2)))
    return float(f32(f32(param) * f32(s)) / f32(n_train))


def regularise(G, lam: float, last_row: bool):
    """add_diag_kernel: G + lambda on the diagonal, one float32 addition per entry (bias row only if last_row)"""
    G = np.array(G, f32)
    D = G.shape[0]
    idx = np.arange(D if last_row else D - 1)
    G[idx, idx] = (G[idx, idx] + f32(lam)).astype(f32)
    return G


def _norm2_spd(A, its=100):
    """largest eigenvalue of a symmetric non-negative matrix, by power iteration"""
    v = np.ones(A.shape[0])
    for _ in range(its):
        v = A @ v
        v /= np.linalg.norm(v)
    return float(v @ A @ v)


class Truth:
    """float64 solution of the regularised float32 system and what its bars need (module docstring)"""

    def __init__(self, Greg, M: int, gram_err=None):
        D = Greg.shape[0]
        full = sym_from_upper(Greg)
        rhs = np.asarray(Greg[:, D:D + M], np.float64)
        p = full[-1, -1]
        s = full[:-1, -1]
        self.p, self.s, self.rb = p, s, rhs[-1]
        self.S = full[:-1, :-1] - np.outer(s, s) / p
        self.b = rhs[:-1] - np.outer(s, rhs[-1]) / p
        self.U = np.linalg.cholesky(self.S).T
        self.Sinv = np.linalg.inv(self.S)
        self.Sinv2 = self.Sinv ** 2
        self.w = sl.cho_solve((self.U, False), self.b)
        self.xb = (rhs[-1] - s @ self.w) / p
        self.UtU = np.abs(self.U.T) @ np.abs(self.U)
        self.Snorm = _norm2_spd(self.S)
        self.gram_err = gram_err
        if gram_err is not None:
            # first-order propagation of the Gram's per-element error E through S = G_ww - s s^T / p and b = R_w - s r_b / p
            E = gram_err
            Es, Ep = E[:-1, D - 1], E[D - 1, D - 1]
            self.ES = E[:-1, :D - 1] + (np.outer(np.abs(s), Es) + np.outer(Es, np.abs(s))) / p + np.outer(np.abs(s), np.abs(s)) * Ep / p ** 2
            self.Eb = E[:-1, D:D + M] + (np.outer(np.abs(s), E[D - 1, D:D + M]) + np.outer(Es, np.abs(rhs[-1]))) / p \
                + np.outer(np.abs(s), np.abs(rhs[-1])) * Ep / p ** 2

    def bar_w(self, mode: int):
        """LAMBDA_RW * sqrt(|S^-1|^2 (tau^2 (|U^T||U|)^2 |w|^2 + tau^2 |b|^2)): the per-entry perturbations are bounded
        deterministically, their signs are independent, so through S^-1 they add as a random walk (module docstring)"""
        D = self.S.shape[0] + 1
        t = tau_entry(mode, D)
        w2 = self.w ** 2
        var = t * t * (self.UtU ** 2 @ w2 + self.b ** 2)
        if self.gram_err is not None:
            var = var + self.ES ** 2 @ w2 + self.Eb ** 2
        return LAMBDA_RW * np.sqrt(self.Sinv2 @ var)

    def bar_xb(self, bar_w):
        """the bias from w: |s|^T bar_w / p, plus its own rounding to float32 and, for the learn path, the Gram's error in s, r_b, p"""
        bar = np.abs(self.s) @ bar_w / self.p + 2 * U * np.abs(self.xb)
        if self.gram_err is not None:
            D = self.S.shape[0] + 1
            E = self.gram_err
            M = self.b.shape[1]
            bar = bar + LAMBDA_RW * (E[D - 1, D:D + M] + E[:-1, D - 1] @ np.abs(self.w) + E[D - 1, D - 1] * np.abs(self.xb)) / self.p
        return bar

    def eta(self, w):
        """normwise backward error of each column of w as a solution of S w = b"""
        w = np.asarray(w, np.float64)
        r = self.b - self.S @ w
        return np.linalg.norm(r, axis=0) / (self.Snorm * np.linalg.norm(w, axis=0) + np.linalg.norm(self.b, axis=0))

    def eta_spotrs(self):
        """eta of LAPACK float32 Cholesky (spotrf + spotrs) on the float32 S and b"""
        S32, b32 = self.S.astype(f32), self.b.astype(f32)
        w = sl.cho_solve(sl.cho_factor(S32, lower=False), b32)
        return self.eta(w.astype(f32))

    def rho(self):
        return float(np.linalg.norm(self.UtU) / np.linalg.norm(self.S))

    def split_can_break(self, mode: int) -> bool:
        """whether the trailing updates' operand split alone (SPLIT_UPDATE[mode] |U^T||U|) can move S's smallest eigenvalue to
        zero: only then may a factorisation in that gram mode report a matrix that is not positive definite"""
        return SPLIT_UPDATE[mode] * self.utu_norm() >= self.smin()

    def smin(self):
        """smallest eigenvalue of S"""
        return 1.0 / _norm2_spd(self.Sinv)

    def utu_norm(self):
        """|| |U^T||U| ||_2"""
        return _norm2_spd(self.UtU)

    def eta_excess(self, mode: int):
        return SPLIT_UPDATE[mode] * self.rho() + U


def ratio(w_got, w_true, bar):
    """|w^ - w| / bar, element by element"""
    return np.abs(np.asarray(w_got, np.float64) - w_true) / np.maximum(bar, 1e-300)


def worst_by_tile(r, rows=PB, cols=64):
    """the worst ratio per (128-row block, 64-column group) of the factorisation's right-hand sides: where a defect sits.  The
    kernels group the columns of Xp = [carried bias column | X], so column c of X is column c + 1 of Xp; the carried column is
    not an output and counts as 0 here, and group g holds X's columns 64 g - 1 .. 64 g + 62"""
    r = np.hstack([np.zeros((r.shape[0], 1)), r])
    nr, nc = -(-r.shape[0] // rows), -(-r.shape[1] // cols)
    out = np.zeros((nr, nc))
    for i in range(nr):
        for j in range(nc):
            out[i, j] = r[i * rows:(i + 1) * rows, j * cols:(j + 1) * cols].max()
    return out


# ---- restatement of cholesky_solve ----------------------------------------------------------------------------------------
def _update(P, arith: str):
    """P^T P as the trailing-update SYRK computes it: 'split' unbiased 3xTF32, 'single' one TF32 pass, 'fp32' SIMT"""
    if arith == "fp32":
        return (P.T @ P).astype(f32)
    if arith == "single":
        T = R.trunc_tf32(P)
        return (T.T @ T).astype(f32)
    hi = R.rna_tf32(P)
    lo = R.rna_tf32((P - hi).astype(f32))
    return ((lo.T @ hi + hi.T @ lo).astype(f32) + (hi.T @ hi).astype(f32)).astype(f32)


def _factor_block(A):
    """U and W = U^-1 of a diagonal block given by its upper triangle, in float32"""
    A = np.triu(A) + np.triu(A, 1).T
    Ub = np.linalg.cholesky(A.astype(f32)).T.astype(f32)
    W = sl.solve_triangular(Ub, np.eye(Ub.shape[0], dtype=f32), lower=False).astype(f32)
    return Ub, W


def cholesky_restated(G, n: int, arith: str = "split", defect=None):
    """solve of the n x n system in the upper triangle of G[:, :n] for the columns G[:, n:], float32.
    defect: ("head" | "tail", panel, row, col) leaves a 64 x 64 tile out of that panel's head / tail update (row, col relative to
    the updated matrix, col >= row); ("fused_row", panel) drops the last row of the A^T P term; ("backsub_w", block) multiplies
    by W^T instead of W in that block of the back substitution"""
    G = np.array(G, f32)
    Ws = {}
    nblocks = -(-n // PB)
    for p, j in enumerate(range(0, n, PANEL)):
        nb1 = min(PB, n - j)
        nb2 = min(PB, n - j - nb1)
        U1, W1 = _factor_block(G[j:j + nb1, j:j + nb1])
        G[j:j + nb1, j:j + nb1] = U1
        Ws[j // PB] = W1
        j3 = j + nb1 + nb2
        if nb2 > 0:
            P1a = (W1.T @ G[j:j + nb1, j + nb1:j3]).astype(f32)
            G[j:j + nb1, j + nb1:j3] = P1a
            A22 = (G[j + nb1:j3, j + nb1:j3] - (P1a.T @ P1a).astype(f32)).astype(f32)
            U2, W2 = _factor_block(A22)
            G[j + nb1:j3, j + nb1:j3] = U2
            Ws[j // PB + 1] = W2
        if G.shape[1] <= j3:
            continue
        P1 = (W1.T @ G[j:j + nb1, j3:]).astype(f32)
        G[j:j + nb1, j3:] = P1
        if nb2 > 0:
            q = nb1 - 1 if defect is not None and defect[0] == "fused_row" and defect[1] == p else nb1
            T = (G[j + nb1:j3, j3:] - (P1a[:q].T @ P1[:q]).astype(f32)).astype(f32)
            G[j + nb1:j3, j3:] = (W2.T @ T).astype(f32)
        rest = n - j3
        if rest <= 0:
            continue
        Pp = G[j:j3, j3:]
        upd = _update(Pp, arith)[:rest]                  # rows of the trailing matrix, every column right of the panel
        head = min(rest, PANEL)
        if defect is not None and defect[0] in ("head", "tail") and defect[1] == p:
            r0, c0 = defect[2], defect[3]
            if defect[0] == "tail":
                r0 += head
                c0 += head
            upd[r0:r0 + 64, c0:c0 + 64] = 0.0
        G[j3:, j3:] = (G[j3:, j3:] - upd).astype(f32)
    X = np.zeros((n, G.shape[1] - n), f32)
    Y = G[:, n:].copy()
    for b in reversed(range(nblocks)):
        r0 = b * PB
        nb = min(PB, n - r0)
        W = Ws[b]
        if defect is not None and defect[0] == "backsub_w" and defect[1] == b:
            W = W.T
        Xb = (W @ Y[r0:r0 + nb]).astype(f32)
        X[r0:r0 + nb] = Xb
        Y[:r0] = (Y[:r0] - (G[:r0, r0:r0 + nb] @ Xb).astype(f32)).astype(f32)
    return X


def solve_gram_restated(G, M: int, reg, n_train: int, arith: str = "split", defect=None, mu=None):
    """sd_solve_gram (D > 256) in numpy: lambda, diagonal, bias-first elimination, cholesky_restated, bias back-substitution.
    reg = (type, param, regularise_last_row).  mu: the column shift of centred rows (sd_learn_centred): lambda is then taken
    from the norm of the uncentred Gram it stands for.  defect, beyond those of cholesky_restated: ("pivot_n_minus_1",) divides
    by p - 1; ("centred_norm",) takes lambda from the centred Gram.  Returns X (D x M), Xc (centred weights) and lambda."""
    G = np.array(G, f32)
    D = G.shape[0]
    typ, param, last_row = reg
    if typ == 1:
        if mu is not None and not (defect is not None and defect[0] == "centred_norm"):
            lam = lambda_matrix_norm(uncentre_gram(G, mu, n_train), param, n_train)
        else:
            lam = lambda_matrix_norm(G, param, n_train)
    else:
        lam = float(f32(param))
    G = regularise(G, lam, last_row)
    sv = np.asarray(G[:, D - 1], np.float64).copy()
    p = sv[D - 1] - (1.0 if defect is not None and defect[0] == "pivot_n_minus_1" else 0.0)
    s = sv[:D - 1]
    rb = np.asarray(G[D - 1, D:D + M], np.float64)
    W = np.zeros((D - 1, D + M), np.float64)
    full_ww = np.triu(np.asarray(G[:D - 1, :D - 1], np.float64))
    W[:, :D - 1] = full_ww - np.triu(np.outer(s, s) / p)
    W[:, D - 1] = s
    W[:, D:] = np.asarray(G[:D - 1, D:D + M], np.float64) - np.outer(s, rb) / p
    Xp = cholesky_restated(W.astype(f32), D - 1, arith, defect if defect is not None and defect[0] not in
                           ("pivot_n_minus_1", "centred_norm") else None)
    w = Xp[:, 1:]
    cprime = (rb - s @ w.astype(np.float64)) / p
    shift = 0.0 if mu is None else np.asarray(mu[:D - 1], np.float64) @ w.astype(np.float64)
    X = np.vstack([w, (cprime - shift).astype(f32)[None]])
    Xc = np.vstack([w, cprime.astype(f32)[None]])
    return X, Xc, lam


def uncentre_gram(Gc, mu, n):
    """the upper triangle of A^T A from the centred Gram, its bias column s' and mu (frob_upper_centred_kernel), float64"""
    D = Gc.shape[0]
    T = sym_from_upper(Gc)
    mu = np.asarray(mu, np.float64).copy()
    mu[D - 1] = 0.0
    sp = T[:, D - 1].copy()
    sp[D - 1] = 0.0
    out = T + np.outer(sp, mu) + np.outer(mu, sp) + n * np.outer(mu, mu)
    out[:D - 1, D - 1] = T[:D - 1, D - 1] + n * mu[:D - 1]
    out[D - 1, :D - 1] = out[:D - 1, D - 1]
    return out


# ---- the learn path ------------------------------------------------------------------------------------------------------
def centre_restated(A, last_row: bool):
    """sd_centre_features on one rank: mu[c] = (float)(column sum in double / N) for the feature columns and 0 for the bias,
    A_c = A - mu by one float32 subtraction per entry -- when D > 256, the last column is exactly ones and it carries no
    penalty; otherwise mu = 0 and A is left as it is"""
    A = np.asarray(A, f32)
    N, D = A.shape
    last = A[:, -1].astype(np.float64)
    mu = np.zeros(D, f32)
    if D > LU_MAX_DIM and not last_row and last.sum() == N and (last * last).sum() == N:
        mu[:-1] = (A[:, :-1].astype(np.float64).sum(axis=0) / N).astype(f32)
    return mu, (A - mu).astype(f32) if mu.any() else A.copy()


def gram_entry_error(Ac, B):
    """the Gram's per-entry error on [A_c^T A_c | A_c^T B] before the random-walk factor: (SPLIT + sqrt(R) u) ||a_i|| ||a_j||
    with gemm_ref's split and rounding counts, gram mode 0 on the tensor cores or the SIMT route, the larger.  Truth.bar_w and
    Truth.bar_xb apply LAMBDA_RW once to it (gemm_ref.gram_bar is this times LAMBDA on its rounding term)"""
    n = Ac.shape[0]
    t0 = R.SPLIT[0] + math.sqrt(R.MMA_STEPS[0] + -(-n // R.KC)) * U
    t2 = math.sqrt(n + 64) * U
    return max(t0, t2) / R.tau_gram(0, n) * R.gram_bar(Ac, B, 0)


def learn_truth(Ac, B, lam: float, last_row: bool):
    """Truth of (A_c^T A_c + Lambda) [w; c'] = A_c^T B in float64 from the float32 rows the Gram reads, with the Gram's bar"""
    G = R.gram_ref(Ac, B)
    D = G.shape[0]
    idx = np.arange(D if last_row else D - 1)
    G[idx, idx] += lam
    return Truth(G, B.shape[1], gram_err=gram_entry_error(Ac, B))


def lambda_bar(A, Ac, mu, param: float):
    """how far lambda = param ||A^T A||_F / N may be from the float64 norm of the float32 A: the centred Gram's bar carried
    through the uncentring (|mu| times the bias column's bar), the rounding of A_c (2u |A|^T |A|), summed into the norm,
    and lambda's own two float32 roundings"""
    N, D = np.asarray(A).shape
    E = R.gram_bar(Ac, None, 0 if R.tau_gram(0, N) >= R.tau_gram(2, N) else 2)
    m = np.abs(np.asarray(mu, np.float64))
    Eb = E[:, D - 1]
    full = E + np.outer(Eb, m) + np.outer(m, Eb) + 2 * U * (np.abs(A.astype(np.float64)).T @ np.abs(A.astype(np.float64)))
    nrm = np.linalg.norm(R.gram_ref(A))
    return param * np.linalg.norm(full) / N + 3 * U * param * nrm / N


# ---- the GPU sweep of sd_solve_gram (tests/test_gpu_cholesky.py); test_chol_bars.py checks the bars on its shapes ----------
# (D, M, cond, gram mode, pitch, regulariser type, regularise_last_row).  D - 1 crosses the 128-block and 256-panel edges
# (256 = one full panel and no trailing matrix, 257 = a one-row ragged block, 384 = a panel with a single block, 4096 = more
# tail tiles than SMs); M + 1 (the bias column rides as right-hand side 0) crosses the 64-column groups (64, 65, 128, 136,
# 137, 192, 193).  pitch (PITCHES): "tight" ldg = D + M, "pad" round4(D + M) + 8, "skew" the same with G's base one float
# off alignment, "odd" an odd ldg.  The trailing updates run on the tensor cores only with an aligned base and ldg % 4 == 0
# (`trailing_routes`): "skew" and "odd" are the deliberate SIMT cases, the "tight" ones have D + M % 4 == 0.  Every gram mode
# 0, 1 and 3 reaches tensor-core head and tail updates at every condition number, and so does every D = 4097 case
# (test_chol_bars.test_sweep_reaches_the_tensor_cores).
SWEEP = [
    (257, 1, 1e1, 0, "tight", 0, 0), (258, 63, 1e3, 0, "odd", 0, 0), (384, 64, 1e5, 0, "skew", 1, 0),
    (385, 127, 1e7, 3, "pad", 0, 1), (386, 136, 1e1, 2, "odd", 0, 0), (512, 192, 1e3, 0, "tight", 1, 1),
    (513, 1, 1e5, 3, "skew", 0, 0), (513, 135, 1e7, 0, "tight", 0, 0), (641, 63, 1e1, 0, "tight", 1, 0),
    (641, 64, 1e5, 2, "tight", 0, 0), (769, 127, 1e3, 3, "tight", 1, 0), (769, 192, 1e7, 0, "skew", 0, 1),
    (1025, 63, 1e1, 1, "tight", 0, 0), (1025, 64, 1e3, 0, "odd", 0, 0), (1025, 136, 1e5, 0, "pad", 1, 0),
    (1025, 1, 1e7, 2, "skew", 0, 0), (1153, 127, 1e3, 2, "odd", 0, 1), (1153, 191, 1e5, 3, "tight", 0, 0),
    (1153, 63, 1e7, 3, "tight", 1, 0), (1537, 63, 1e7, 1, "tight", 0, 0), (2049, 135, 1e1, 0, "tight", 1, 0),
    (2049, 64, 1e3, 1, "pad", 0, 0), (2049, 192, 1e5, 0, "skew", 0, 0), (2049, 63, 1e7, 0, "tight", 0, 0),
    (2049, 1, 1e3, 3, "odd", 0, 0), (2600, 136, 1e3, 0, "odd", 0, 0), (2600, 64, 1e5, 2, "tight", 1, 0),
    (2600, 127, 1e5, 1, "pad", 0, 1), (4097, 135, 1e3, 0, "tight", 1, 0), (4097, 192, 1e5, 3, "pad", 0, 0),
    (4097, 63, 1e1, 3, "tight", 0, 0),
]


def pitch(kind: str, w: int):
    """(ldg, shift of G's base in floats) of a pitch kind for rows of w = D + M floats"""
    if kind == "tight":
        return w, 0
    if kind == "odd":
        return (w + 1) | 1, 0
    return (w + 3) // 4 * 4 + 8, (1 if kind == "skew" else 0)


def trailing_routes(D: int, M: int, mode: int, ldg: int, aligned: bool):
    """for each panel of cholesky_solve that has a trailing matrix: (tensor cores?, has a tail update?).  syrk_upper takes the
    tensor cores when syrk_is_big(K, rows, columns) holds for the whole update, the gram mode is not 2 and TMA can read the
    panel rows (16-byte aligned base, ldg % 4 == 0); the head and the tail of one panel take the same route"""
    n, out = D - 1, []
    for j in range(0, n, PANEL):
        nb1 = min(PB, n - j)
        nb2 = min(PB, n - j - nb1)
        j3 = j + nb1 + nb2
        rest, cols3 = n - j3, D + M - j3
        if rest <= 0:
            continue
        big = rest * cols3 >= 256 * 256 and nb1 + nb2 >= 64
        out.append((big and mode != 2 and aligned and ldg % 4 == 0 and (j * ldg + j3) % 4 == 0, rest > PANEL))
    return out


GUARD_ROWS = 2                              # rows of sentinels before and after G in the GPU test's buffer


def g_offset(ldg: int, shift: int) -> int:
    """floats from the start of the GPU test's buffer (a 16-byte aligned allocation) to G's first entry"""
    return GUARD_ROWS * ldg + shift


def case_routes(c):
    """trailing_routes of a sweep case laid out as the GPU test lays it out"""
    D, M, _, mode, kind, _, _ = c
    ldg, shift = pitch(kind, D + M)
    return trailing_routes(D, M, mode, ldg, g_offset(ldg, shift) % 4 == 0)


def syrk_launches(routes):
    """(tensor-core, SIMT) SYRK launches of one factorisation: a head update per panel, a tail update when there is one"""
    tc = sum(1 + tail for t, tail in routes if t)
    return tc, sum(1 + tail for t, tail in routes if not t)


LAMBDA_DESIGN = 1e-3                        # the lambda every designed system is built around
N_DESIGN = 1000                             # its bias pivot p = sample count


def sweep_id(c):
    D, M, cond, mode, pitch, typ, last = c
    return f"D{D}-M{M}-cond{cond:.0e}-mode{mode}-{pitch}-{'norm' if typ else 'manual'}-last{last}"


def sweep_system(c):
    """the float32 [G | R] of a sweep case and the regulariser (type, param, last_row) that gives it lambda ~ LAMBDA_DESIGN"""
    D, M, cond, mode, pitch, typ, last = c
    G = designed_gram(D, M, cond, LAMBDA_DESIGN, bool(last), seed=D * 1000 + M)
    param = LAMBDA_DESIGN
    if typ == 1:
        param = LAMBDA_DESIGN * N_DESIGN / np.linalg.norm(sym_from_upper(G))
    return G, (typ, float(f32(param)), last)


# ---- systems of a given condition number ----------------------------------------------------------------------------------
_Q = {}


def orthogonal(n: int):
    if n not in _Q:
        _Q[n] = np.linalg.qr(np.random.default_rng(n).standard_normal((n, n)))[0]
    return _Q[n]


def designed_gram(D: int, M: int, cond: float, lam: float, last_row: bool, seed: int, n_samples: int = 1000,
                  coupling: float = 0.0025):
    """a float32 [G | R] (D x (D + M), full) whose regularised, bias-eliminated system S has the float64 spectrum
    logspace(0, -log10(cond)) before rounding: G_ww = S + s s^T / p - lambda I, pivot p = n_samples (a sample count), bias
    column s = p * mean with means up to sqrt(coupling) (s s^T / p is at most coupling: small enough that rounding G_ww to
    float32 keeps the designed spectrum at 1e7), right-hand sides of unit size"""
    rng = np.random.default_rng(seed)
    n = D - 1
    Q = orthogonal(n)
    S = (Q * np.logspace(0, -math.log10(cond), n)) @ Q.T
    p = float(n_samples)
    s = p * math.sqrt(coupling / p) * rng.random(n)
    G = np.zeros((D, D + M))
    G[:n, :n] = S + np.outer(s, s) / p - lam * np.eye(n)
    G[:n, n] = s
    G[n, :n] = s
    G[n, n] = p - (lam if last_row else 0.0)
    G[:, D:] = rng.standard_normal((D, M))
    G[:, :D] = (G[:, :D] + G[:, :D].T) / 2
    return G.astype(f32)


# ---- restatement of lu_small_kernel ---------------------------------------------------------------------------------------
def lu_restated(G, M: int):
    """lu_small_kernel on the float32 D x (D + M) matrix G (upper triangle and right-hand sides read): mirror the upper
    triangle, pivot on the first largest |G[i][k]| in ascending row order, swap rows over all D + M columns, multipliers by one
    division, trailing update with the product and the difference rounded separately (rows with a zero multiplier skipped), back
    substitution in ascending k, one division.  Returns X (D x M) and whether a zero pivot was met."""
    G = np.array(G, f32)
    D = G.shape[0]
    iu = np.triu_indices(D, 1)
    G[iu[1], iu[0]] = G[iu]
    singular = False
    for k in range(D):
        col = np.abs(G[k:, k])
        piv = k + int(np.argmax(col))
        if not (col[piv - k] > 0):
            singular = True
        if piv != k:
            G[[k, piv]] = G[[piv, k]]
        with np.errstate(all="ignore"):
            L = (G[k + 1:, k] / G[k, k]).astype(f32)
            G[k + 1:, k] = L
            prod = (L[:, None] * G[k, k + 1:][None, :]).astype(f32)
            G[k + 1:, k + 1:] = np.where((L != 0)[:, None], (G[k + 1:, k + 1:] - prod).astype(f32), G[k + 1:, k + 1:])
    X = G[:, D:D + M].copy()
    with np.errstate(all="ignore"):
        for i in range(D - 1, -1, -1):
            r = X[i].copy()
            for k in range(i + 1, D):
                r = (r - (G[i, k] * X[k]).astype(f32)).astype(f32)
            X[i] = (r / G[i, i]).astype(f32)
    return X, singular
