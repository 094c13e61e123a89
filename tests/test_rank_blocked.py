"""The rank diagnostic's algorithm (superviseddescent_b200/csrc/sd_rank.cu) restated in float64, without a GPU.

The device routine is a blocked, right-looking, diagonally pivoted Cholesky without row or column swaps: panels of nb pivots,
each pivot the largest live Schur-complement diagonal (ties: the smallest index), chosen indices marked dead with zero factor
entries, the trailing update over the whole matrix (dead rows included), and a stop at the first pivot <= eps_f32 * D * d0 or
<= 0.  Here that restatement must give the rank LAPACK's dpstrf gives at the same tolerance, and the pivot sequence of the
unblocked, left-looking form it replaced (dpstrf swaps rows, so its tie order is not this one)."""
import numpy as np
import pytest
from scipy.linalg import lapack

EPS_F32 = float(np.finfo(np.float32).eps)


def blocked_rank(G, nb=128):
    """The device algorithm: upper triangle only, panels of nb pivots, full-matrix trailing update."""
    D = G.shape[0]
    C = np.triu(G).astype(np.float64)
    dwork = np.diag(G).astype(np.float64).copy()          # -1: chosen
    thr = EPS_F32 * D
    rank, d0, pivots = 0, None, []
    while rank < D:
        Lt = np.zeros((nb, D))
        k, stop = 0, False
        while k < nb and rank + k < D:
            p = int(np.argmax(dwork))                     # first maximum: the smallest index wins a tie
            pv = dwork[p]
            if rank + k == 0:
                d0 = pv
            if not (pv > thr * d0) or not (pv > 0):
                stop = True
                break
            r = np.sqrt(pv)
            col = np.concatenate([C[:p + 1, p], C[p, p + 1:]]) - Lt[:k].T @ Lt[:k, p]
            live = dwork >= 0
            l = np.where(live, col / r, 0.0)
            l[p] = r
            Lt[k] = l
            dwork = np.where(live, np.maximum(dwork - l * l, 0.0), dwork)
            dwork[p] = -1.0
            pivots.append(p)
            k += 1
        rank += k
        if stop or rank == D:
            break
        C -= np.triu(Lt[:k].T @ Lt[:k])
    return rank, pivots


def unblocked_rank(G):
    """The one-CTA kernel the blocked routine replaced: left-looking, column p of G minus all earlier factor rows."""
    D = G.shape[0]
    U = np.triu(G).astype(np.float64)
    dwork = np.diag(G).astype(np.float64).copy()
    L = np.zeros((D, D))
    thr = EPS_F32 * D
    d0, pivots = None, []
    for k in range(D):
        p = int(np.argmax(dwork))
        pv = dwork[p]
        if k == 0:
            d0 = pv
        if not (pv > thr * d0) or not (pv > 0):
            break
        r = np.sqrt(pv)
        col = np.concatenate([U[:p + 1, p], U[p, p + 1:]]) - L[:k].T @ L[:k, p]
        live = dwork >= 0
        l = np.where(live, col / r, 0.0)
        l[p] = r
        L[k] = l
        dwork = np.where(live, np.maximum(dwork - l * l, 0.0), dwork)
        dwork[p] = -1.0
        pivots.append(p)
    return len(pivots), pivots


def dpstrf_rank(G):
    D = G.shape[0]
    tol = EPS_F32 * D * float(np.max(np.diag(G)))
    _, _, rank, info = lapack.dpstrf(np.array(G, dtype=np.float64, order="F"), tol=tol, lower=0)
    assert info in (0, 1)
    return int(rank)


def check(G, nb=128, expect=None, same_order=True):
    rb, pb = blocked_rank(G, nb)
    ru, pu = unblocked_rank(G)
    if same_order:
        assert pb == pu, "pivot sequences differ"
    assert rb == ru == dpstrf_rank(G)
    if expect is not None:
        assert rb == expect
    return rb


def low_rank_gram(rng, D, r):
    X = rng.standard_normal((r, D))
    return X.T @ X


def test_partial_last_panel_full_rank():
    """D = 700 = 5 x 128 + 60: the last panel stops at D, not at nb."""
    rng = np.random.default_rng(1)
    X = rng.standard_normal((1000, 700))
    check(X.T @ X + np.eye(700), expect=700)


@pytest.mark.parametrize("r", [1, 127, 128, 129, 300, 450])
def test_random_psd_of_known_rank(r):
    check(low_rank_gram(np.random.default_rng(r), 700, r), expect=r)


@pytest.mark.parametrize("nb", [1, 7, 64, 128, 1024])
def test_panel_width_does_not_change_the_answer(nb):
    G = low_rank_gram(np.random.default_rng(5), 300, 211)
    assert blocked_rank(G, nb) == unblocked_rank(G)


def test_duplicated_columns():
    """40 duplicated feature columns and a bias column of ones, lambda = 0: rank D - 40."""
    rng = np.random.default_rng(2)
    A = rng.random((1000, 300))
    A[:, -1] = 1.0
    A[:, 10:50] = A[:, 100:140]
    check(A.T @ A, expect=260)
    # the same with lambda > 0 on the diagonal is regular.  The duplicates' last pivots are then all about lambda and tie up to
    # rounding, so the two forms may take them in another order: only the rank is compared.
    check(A.T @ A + 0.5 * np.eye(300), expect=300, same_order=False)


def test_exact_ties_take_the_smallest_index():
    """Identical 2 x 2 blocks [[4, 2], [2, 4]]: every first pivot ties at 4 and the downdate leaves exactly 3, so the order is
    0, 2, 4, ... then 1, 3, 5, ... -- across panel boundaries (nb = 7)."""
    n = 40
    G = np.kron(np.eye(n // 2), np.array([[4.0, 2.0], [2.0, 4.0]]))
    rank, piv = blocked_rank(G, nb=7)
    assert rank == n
    assert piv == list(range(0, n, 2)) + list(range(1, n, 2))
    check(G, nb=7, expect=n)
    # a diagonal matrix with repeated values: ties broken by index, zeros stop the factorisation
    d = np.array([3.0, 5.0, 5.0, 0.0, 3.0, 5.0, 0.0, 1.0])
    rank, piv = blocked_rank(np.diag(d), nb=3)
    assert rank == 6 and piv == [1, 2, 5, 0, 4, 7]
    check(np.diag(d), nb=3, expect=6)


def test_zero_matrix_has_rank_zero():
    assert blocked_rank(np.zeros((5, 5)))[0] == 0
