"""The acceptance checks of tests/la_checks.py on CPU: each passes a correct NumPy result and fails one with a
single injected defect of the kind a kernel could have.  No GPU needed."""

import re

import numpy as np
import pytest
import scipy.linalg

import la_checks as lc


def _spd(n, seed):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n, n))
    return G @ G.T / n + np.eye(n)


def test_gamma_and_unit_roundoff():
    assert lc.U == np.finfo(np.float64).eps / 2
    assert lc.gamma(1) > lc.U and lc.gamma(1000) > 1000 * lc.U


def test_padding_check_bitwise():
    rng = np.random.default_rng(0)
    A = rng.standard_normal((20, 13))
    before = lc.with_padding(A, 16)
    after = before.copy()
    after[:, :13] += 1.0  # the defined columns may change
    lc.check_padding_unchanged(before, after, 13)
    bad = after.copy()
    bad[7, 14] = 0.0  # one padding column written
    with pytest.raises(AssertionError, match='padding columns'):
        lc.check_padding_unchanged(before, bad, 13)
    other_nan = after.copy()
    other_nan.view(np.uint64)[3, 15] ^= 1  # another NaN payload is a write too
    assert np.isnan(other_nan[3, 15])
    with pytest.raises(AssertionError):
        lc.check_padding_unchanged(before, other_nan, 13)


def test_gram_check():
    rng = np.random.default_rng(1)
    X = rng.standard_normal((300, 40))
    lam = 1e-3
    C = lc.with_padding(X.T @ X + lam * np.eye(40), 42)
    C[np.triu_indices(40, 1)] = np.nan  # upper triangle is not part of the result
    lc.check_gram(X, C, lam)
    bad = C.copy()
    bad[17, 17] -= lam  # lam missing from one diagonal entry
    with pytest.raises(AssertionError, match='gram_tn'):
        lc.check_gram(X, bad, lam)
    nan = C.copy()
    nan[30, 2] = np.nan
    with pytest.raises(AssertionError):
        lc.check_gram(X, nan, lam)


def _dropped_row_sum(X, v, drop=1):
    """X^T v with row `drop` left out (what a 256-row chunk that loses one row produces)."""
    keep = np.ones(X.shape[0], dtype=bool)
    keep[drop] = False
    return X[keep].T @ v[keep]


def test_project_and_sqnorm_checks():
    rng = np.random.default_rng(2)
    X = rng.standard_normal((600, 33))
    v = rng.standard_normal(600)
    lc.check_project(X, v, X.T @ v)
    with pytest.raises(AssertionError, match='nystroem_project'):
        lc.check_project(X, v, _dropped_row_sum(X, v))  # one row of a 256-row chunk dropped
    lc.check_row_sqnorms(X, np.sum(X * X, axis=1))
    bad = np.sum(X[:, 1:] ** 2, axis=1)  # one column of every row dropped
    with pytest.raises(AssertionError, match='row_sqnorms'):
        lc.check_row_sqnorms(X, bad)


def test_expand_and_apply_checks():
    rng = np.random.default_rng(3)
    X = rng.standard_normal((700, 97)) * 0.1
    v = rng.standard_normal(700)
    lam = 1e-2
    t = X.T @ v
    lc.check_expand(X, t, v, lam, (X @ t - v) / lam)
    lc.check_apply(X, v, lam, (X @ (X.T @ v) - v) / lam)
    t_bad = _dropped_row_sum(X, v, drop=300)
    with pytest.raises(AssertionError, match='nystroem_apply'):
        lc.check_apply(X, v, lam, (X @ t_bad - v) / lam)
    with pytest.raises(AssertionError, match='nystroem_expand'):
        lc.check_expand(X, t, v, lam, (X @ t - v) / (lam * (1 + 1e-9)))


def test_trsm_check():
    m, n = 300, 50  # three 128-column blocks, the last one partial
    L = np.linalg.cholesky(_spd(m, 4))
    X0 = np.random.default_rng(5).standard_normal((n, m))
    X = scipy.linalg.solve_triangular(L, X0.T, lower=True).T
    Lc = lc.nan_upper(L, m + 2)
    lc.check_trsm_right_lt(Lc[:, :m], X0, lc.with_padding(X, m + 2), cond_ok=True)
    bad = X.copy()
    bad[:, 256:] = X0[:, 256:]  # the last column block left unsolved
    with pytest.raises(AssertionError, match='trsm_right_lt residual'):
        lc.check_trsm_right_lt(Lc[:, :m], X0, bad)
    # an L whose strictly upper triangle was used: with the symmetric values there, and with the NaN canaries
    full = np.tril(L) + np.tril(L, -1).T
    used_upper = np.linalg.solve(full, X0.T).T  # X full^T = X0
    with pytest.raises(AssertionError, match='trsm_right_lt residual'):
        lc.check_trsm_right_lt(L, X0, used_upper)
    with np.errstate(invalid='ignore'):
        nan_used = X0 @ np.where(np.isnan(Lc[:, :m]), np.nan, 0.0)
    with pytest.raises(AssertionError, match='non-finite'):
        lc.check_trsm_right_lt(L, X0, nan_used)


def test_potrs_check():
    n = 200
    A = _spd(n, 6)
    L = np.linalg.cholesky(A)
    B = np.random.default_rng(7).standard_normal((n, 3))
    X = scipy.linalg.cho_solve((L, True), B)
    lc.check_potrs(A, L, B, X, cond_ok=True)
    bad = X.copy()
    bad[128:, 1] = scipy.linalg.solve_triangular(L, B[:, 1], lower=True)[128:]  # last block of the backward sweep skipped
    with pytest.raises(AssertionError, match='potrs residual'):
        lc.check_potrs(A, L, B, bad)


def test_cholesky_check():
    n = 260
    A = _spd(n, 8)
    L = np.linalg.cholesky(A)
    Lc = lc.nan_upper(L, n + 1)
    lc.check_cholesky(A, Lc, forward_tol=1e-12)
    no_lam = _spd(n, 8)
    no_lam[100, 100] -= 1e-6  # a diagonal entry without its shift
    with pytest.raises(AssertionError, match='backward error'):
        lc.check_cholesky(A, np.linalg.cholesky(no_lam))
    used_upper = Lc.copy()
    used_upper[200:, 150] = np.nan  # what reading the NaN canaries of the upper triangle leaves behind
    with pytest.raises(AssertionError, match='non-finite'):
        lc.check_cholesky(A, used_upper)


# ------------------------------------------------------------------------------------------------ GEMM
def _gemm_case(seed=9, m=257, n=257, k=66):
    """Standard-normal operands with rows scaled by 2^e, e in [-20, 20]; C0 at the scale of the product.  Row 9 of A
    and row 5 of B carry 2^-20 and row 0 of each 2^20, so entry (9, 5) is 2^-80 of the largest."""
    rng = np.random.default_rng(seed)
    ea, eb = rng.integers(-20, 21, size=m), rng.integers(-20, 21, size=n)
    ea[[0, 9]] = [20, -20]
    eb[[0, 5]] = [20, -20]
    A = np.ldexp(rng.standard_normal((m, k)), ea[:, None])
    B = np.ldexp(rng.standard_normal((n, k)), eb[:, None])
    C0 = np.ldexp(rng.standard_normal((m, n)) * np.sqrt(k), ea[:, None] + eb[None, :])
    return A, B, C0


def test_gemm_check_accepts_an_independent_evaluation():
    """Extended precision, the k sum taken backwards, rounded once: inside the bound in both forms, with the upper
    triangle NaN under tri, and with NaN in C0 when beta == 0."""
    A, B, C0 = _gemm_case()
    P = A[:, ::-1].astype(np.longdouble) @ B[:, ::-1].T.astype(np.longdouble)
    lc.check_gemm_nt(A, B, C0, (P + C0).astype(np.float64))
    lc.check_gemm_nt(A, B, C0, (0.75 * P - 1.25 * C0).astype(np.float64), alpha=0.75, beta=-1.25)
    lc.check_gemm_nt(A, B, None, P.astype(np.float64), beta=0.0)
    upper_nan = (P + C0).astype(np.float64)
    upper_nan[np.triu_indices(A.shape[0], 1)] = np.nan
    lc.check_gemm_nt(A, B, C0, upper_nan, tri=True)
    with pytest.raises(AssertionError, match='gemm_nt'):
        lc.check_gemm_nt(A, B, C0, upper_nan)


def _gemm_defects():
    A, B, C0 = _gemm_case()
    good = A @ B.T + C0
    out = {}
    d = good.copy()
    d[128:256, :128] = A[128:256, :-4] @ B[:128, :-4].T + C0[128:256, :128]
    out['last k-step dropped in tile (1, 0)'] = (d, '(1, 0)')
    d = good.copy()
    d[136:144, 8:16] = good[136:144, 8:16].T
    out['fragment transposed'] = (d, '(1, 0)')
    d = good.copy()
    d[16:24, 128:136] = C0[16:24, 128:136]
    out['stale fragment'] = (d, '(0, 1)')
    d = good.copy()
    d[:, -1] = C0[:, -1]
    out['last column of an odd n not stored'] = (d, '(0, 2)')
    d = good.copy()
    d[128:256, 128:256] += A[128:256] @ B[128:256].T
    out['tile accumulated twice'] = (d, '(1, 1)')
    out['beta = 0 applied to the accumulating form'] = (A @ B.T, '(0, 0)')
    d = good.copy()
    d[9, 5] = -d[9, 5]
    out['wrong sign in a small row'] = (d, '(0, 0); first at (9, 5)')
    return A, B, C0, good, out


_GEMM_DEFECTS = ['last k-step dropped in tile (1, 0)', 'fragment transposed', 'stale fragment',
                 'last column of an odd n not stored', 'tile accumulated twice',
                 'beta = 0 applied to the accumulating form', 'wrong sign in a small row']


@pytest.mark.parametrize('defect', _GEMM_DEFECTS)
def test_gemm_check_rejects(defect):
    """One defect of the kind a tiled kernel could have, in the accumulating form C0 + A B^T: the check fails and
    names the tile."""
    A, B, C0, good, defects = _gemm_defects()
    assert sorted(defects) == sorted(_GEMM_DEFECTS)
    lc.check_gemm_nt(A, B, C0, good)
    bad, where = defects[defect]
    with pytest.raises(AssertionError, match='gemm_nt: .* in tiles ' + re.escape(where)):
        lc.check_gemm_nt(A, B, C0, bad)
    if defect != 'wrong sign in a small row':
        return
    with pytest.raises(AssertionError):  # (9, 5) is below the diagonal
        lc.check_gemm_nt(A, B, C0, bad, tri=True)
    nan = good.copy()
    nan[200, 3] = np.nan
    with pytest.raises(AssertionError, match=r'tiles \(1, 0\)'):
        lc.check_gemm_nt(A, B, C0, nan, tri=True)


def test_gemm_max_norm_check_misses_what_the_componentwise_bound_sees():
    """max|err| / max|ref| < 1e-13, the assertion of the older GEMM tests, accepts a wrong sign in an entry that is
    2^-80 of the largest; the componentwise bound does not."""
    A, B, C0, good, defects = _gemm_defects()
    bad, _ = defects['wrong sign in a small row']
    assert np.max(np.abs(bad - good)) / np.max(np.abs(good)) < 1e-13
    with pytest.raises(AssertionError):
        lc.check_gemm_nt(A, B, C0, bad)
