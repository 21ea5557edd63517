"""Acceptance checks for the dense linear-algebra building blocks (csrc/solve.cu, csrc/nystroem.cu).

Plain functions on NumPy arrays, shared by the GPU tests (tests/test_dense_la.py, tests/test_gemm_classes.py) and by a CPU test that shows
every check can fail (tests/test_la_checks.py).  Each check raises AssertionError with a short diagnosis.

Bounds are componentwise wherever standard error analysis gives one, with u = 2^-53 and
gamma_k = k u / (1 - k u).  They hold for any summation order, so a tensor-core kernel and NumPy's BLAS both
meet them; the factor 2 in the inner-product bounds covers the rounding of the FP64 NumPy reference itself.
A NaN anywhere in a checked region fails the check (NaN <= bound is false).
"""

import numpy as np

U = 2.0 ** -53


def gamma(k):
    k = max(int(k), 1)
    return k * U / (1.0 - k * U)


def _within(err, bound, what):
    err = np.asarray(err, dtype=np.float64)
    bound = np.asarray(bound, dtype=np.float64)
    ok = err <= bound
    if not np.all(ok):
        bad = np.argwhere(~ok)
        i = tuple(bad[0]) if bad.ndim > 1 and bad.shape[1] else ()
        raise AssertionError(
            '%s: %d entries outside the bound; first at %s: error %r > bound %r'
            % (what, int(bad.shape[0]), i, float(err[i]) if err.ndim else float(err), float(np.broadcast_to(bound, err.shape)[i]))
        )


# ------------------------------------------------------------------------------------------------ canaries
def with_padding(A, ld, fill=np.nan):
    """Copy of A (rows x width) in a (rows x ld) buffer whose padding columns hold `fill`."""
    A = np.asarray(A, dtype=np.float64)
    out = np.full((A.shape[0], ld), fill)
    out[:, : A.shape[1]] = A
    return out


def nan_upper(L, ld=None):
    """Lower-triangular L in a (n x ld) buffer with NaN in the strictly upper triangle and in the padding."""
    n = L.shape[0]
    out = with_padding(np.tril(L), n if ld is None else ld)
    out[np.triu_indices(n, 1)] = np.nan
    return out


def check_padding_unchanged(before, after, width, what='padding'):
    """Columns width..ld-1 of `after` are bit-identical to `before` (NaN payloads included)."""
    b = np.ascontiguousarray(np.asarray(before, dtype=np.float64)[:, width:]).view(np.uint64)
    a = np.ascontiguousarray(np.asarray(after, dtype=np.float64)[:, width:]).view(np.uint64)
    if not np.array_equal(a, b):
        cols = sorted(set(np.argwhere(a != b)[:, 1] + width))
        raise AssertionError('%s: padding columns %s were written' % (what, cols[:8]))


def check_finite(X, what='result'):
    X = np.asarray(X)
    if not np.all(np.isfinite(X)):
        raise AssertionError('%s: %d non-finite entries (first at %s)' % (what, int(np.sum(~np.isfinite(X))), tuple(np.argwhere(~np.isfinite(X))[0])))


# ------------------------------------------------------------------------------------------------ inner products
def check_gram(X, C_hat, lam):
    """C = X^T X + lam I, lower triangle only: |C^ - C| <= 2 gamma_{k+1} (|X|^T |X| + lam I), k = rows of X
    (one extra rounding for adding lam)."""
    X = np.asarray(X, dtype=np.float64)
    m = X.shape[1]
    C_hat = np.asarray(C_hat, dtype=np.float64)[:m, :m]
    ref = X.T @ X + lam * np.eye(m)
    bound = 2 * gamma(X.shape[0] + 1) * (np.abs(X).T @ np.abs(X) + abs(lam) * np.eye(m))
    low = np.tril_indices(m)
    check_finite(C_hat[low], 'gram lower triangle')
    _within(np.abs(C_hat - ref)[low], bound[low], 'gram_tn')


GEMM_TILE = 128  # tile edge of the DMMA GEMM kernels (csrc/solve.cu); failures are reported by tile


def tiles_of(bad, limit=6):
    """'(ti, tj), ...' of the GEMM tiles that hold a True entry of the boolean matrix `bad`."""
    idx = np.argwhere(bad)
    tiles = sorted(set(map(tuple, (idx // GEMM_TILE).tolist())))
    return ', '.join('(%d, %d)' % t for t in tiles[:limit]) + (' and %d more' % (len(tiles) - limit) if len(tiles) > limit else '')


def check_gemm_nt(A, B, C0, C_hat, alpha=1.0, beta=1.0, tri=False, what='gemm_nt'):
    """C = alpha A B^T + beta C0 with A (m x k), B (n x k), componentwise:
    |C^ - C| <= 2 gamma_{k+2} (|alpha| |A| |B|^T + |beta| |C0|).
    The k products and k - 1 additions of an entry, in any order, carry gamma_k; scaling by alpha, scaling C0 by beta
    and adding the two give gamma_{k+2}.  The accumulating form C0 + A B^T (accumulators that start from C0: k
    additions, no scaling) is alpha = beta = 1 and lies inside the same bound.  C0 may be None when beta == 0.
    tri: only entries with col <= row are part of the result."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    m, k = A.shape
    n = B.shape[0]
    C_hat = np.asarray(C_hat, dtype=np.float64)[:m, :n]
    ref = alpha * (A @ B.T)
    bound = abs(alpha) * (np.abs(A) @ np.abs(B).T)
    if beta != 0.0:
        C0 = np.asarray(C0, dtype=np.float64)[:m, :n]
        ref += beta * C0
        bound += abs(beta) * np.abs(C0)
    bound *= 2 * gamma(k + 2)
    with np.errstate(invalid='ignore'):
        err = np.abs(C_hat - ref)
        bad = ~(err <= bound)  # NaN fails
    if tri:
        bad &= np.tri(m, n, dtype=bool)
    if bad.any():
        r, c = np.argwhere(bad)[0]
        raise AssertionError(
            '%s: %d entries outside the bound, in tiles %s; first at (%d, %d): %r, expected %r, error %.3e > bound %.3e'
            % (what, int(bad.sum()), tiles_of(bad), r, c, float(C_hat[r, c]), float(ref[r, c]), float(err[r, c]), float(bound[r, c]))
        )


def check_row_sqnorms(X, out):
    """out[r] = |X[r, :]|^2: |out^ - out| <= 2 gamma_m sum_j X[r, j]^2."""
    X = np.asarray(X, dtype=np.float64)
    ref = np.einsum('ij,ij->i', X, X)
    _within(np.abs(np.asarray(out) - ref), 2 * gamma(X.shape[1]) * ref, 'row_sqnorms')


def check_project(X, v, t):
    """t = X^T v: |t^ - t| <= 2 gamma_n |X|^T |v|, n = rows of X."""
    X = np.asarray(X, dtype=np.float64)
    ref = X.T @ v
    _within(np.abs(np.asarray(t) - ref), 2 * gamma(X.shape[0]) * (np.abs(X).T @ np.abs(v)), 'nystroem_project')


def check_expand(X, t, v, lam, out):
    """out = (X t - v) / lam with t given.

    The row dot product s = X[r, :] t carries at most gamma_m (|X| |t|)[r]; the subtraction s - v adds one
    rounding of |s| + |v|, and the scaling by 1/lam (a rounded reciprocal times a rounded product) two more of the
    result.  So each of the kernel and the reference is within gamma_{m+3} (|X| |t| + |v|) / lam of the exact
    value, and |out^ - out_ref| <= 2 gamma_{m+3} (|X| |t| + |v|) / lam."""
    X = np.asarray(X, dtype=np.float64)
    ref = (X @ t - v) / lam
    bound = 2 * gamma(X.shape[1] + 3) * (np.abs(X) @ np.abs(t) + np.abs(v)) / lam
    _within(np.abs(np.asarray(out) - ref), bound, 'nystroem_expand')


def check_apply(X, v, lam, out):
    """out = (X (X^T v) - v) / lam.

    t^ = X^T v is within gamma_n |X|^T |v| of t (n rows); that error reaches out through X as
    gamma_n |X| (|X|^T |v|) / lam.  The expand step on t^ adds gamma_{m+3} (|X| |t^| + |v|) / lam (check_expand),
    and |t^| <= (1 + gamma_n) |X|^T |v|.  Together, for kernel and reference:
    |out^ - out_ref| <= 2 gamma_{n+m+4} (|X| (|X|^T |v|) + |v|) / lam."""
    X = np.asarray(X, dtype=np.float64)
    ref = (X @ (X.T @ v) - v) / lam
    absX = np.abs(X)
    bound = 2 * gamma(X.shape[0] + X.shape[1] + 4) * (absX @ (absX.T @ np.abs(v)) + np.abs(v)) / lam
    _within(np.abs(np.asarray(out) - ref), bound, 'nystroem_apply')


# ------------------------------------------------------------------------------------------------ triangular solves
TRSM_C = 8
POTRS_C = 8


def check_trsm_right_lt(L, X0, X_hat, cond_ok=False):
    """X^ = X0 L^-T for lower-triangular L (m x m), by its residual:
    |X^ L^T - X0| <= c m u (|X^| |L|^T), c = TRSM_C (a triangular solve is componentwise backward stable; the
    constant also covers the rounding of the residual product).  Only the lower triangle of L is used.
    cond_ok: L is well conditioned, so X^ must also match scipy's solve_triangular to 1e-12 (relative to max|X|)."""
    import scipy.linalg

    Lt = np.tril(np.asarray(L, dtype=np.float64))
    m = Lt.shape[0]
    X_hat = np.asarray(X_hat, dtype=np.float64)[:, :m]
    check_finite(X_hat, 'trsm_right_lt result')
    R = X_hat @ Lt.T - X0
    _within(np.abs(R), TRSM_C * m * U * (np.abs(X_hat) @ np.abs(Lt).T), 'trsm_right_lt residual')
    if cond_ok:
        ref = scipy.linalg.solve_triangular(Lt, np.asarray(X0).T, lower=True, check_finite=False).T  # L X^T = X0^T
        err = np.max(np.abs(X_hat - ref)) / max(np.max(np.abs(ref)), 1e-300)
        if not err <= 1e-12:
            raise AssertionError('trsm_right_lt: %.3e from solve_triangular (> 1e-12)' % err)


def check_potrs(A, L, B0, X_hat, cond_ok=False):
    """X^ = A^-1 B0 from the Cholesky factor L of A, column by column by the residual:
    ||A x^ - b||_inf <= c n u ||A||_inf ||x^||_inf, c = POTRS_C.
    cond_ok: A well conditioned, so X^ must also match scipy's cho_solve (with L) to 1e-12."""
    import scipy.linalg

    A = np.asarray(A, dtype=np.float64)
    n = A.shape[0]
    B0 = np.asarray(B0, dtype=np.float64).reshape(n, -1)
    X_hat = np.asarray(X_hat, dtype=np.float64).reshape(n, -1)[:, : B0.shape[1]]
    check_finite(X_hat, 'potrs result')
    res = np.max(np.abs(A @ X_hat - B0), axis=0)
    bound = POTRS_C * n * U * np.max(np.sum(np.abs(A), axis=1)) * np.max(np.abs(X_hat), axis=0)
    _within(res, bound, 'potrs residual')
    if cond_ok:
        ref = scipy.linalg.cho_solve((np.tril(L), True), B0, check_finite=False)
        err = np.max(np.abs(X_hat - ref)) / max(np.max(np.abs(ref)), 1e-300)
        if not err <= 1e-12:
            raise AssertionError('potrs: %.3e from cho_solve (> 1e-12)' % err)


# ------------------------------------------------------------------------------------------------ Cholesky
def cholesky_backward_error(A, L):
    Lt = np.tril(L)
    return float(np.linalg.norm(A - Lt @ Lt.T) / np.linalg.norm(A))


def check_cholesky(A, L_hat, L_ref=None, forward_tol=None):
    """A = L^ L^T with L^ the lower triangle of L_hat (its strictly upper triangle is not part of the result):
    ||A - L^ L^^T||_F / ||A||_F <= max(8 * the same backward error of LAPACK's factor, 64 n u).
    L_ref: LAPACK's factor (computed here if None).  forward_tol: when A is well conditioned, also
    max|L^ - L_ref| <= forward_tol * max|L_ref|."""
    import scipy.linalg

    A = np.asarray(A, dtype=np.float64)
    n = A.shape[0]
    L_hat = np.tril(np.asarray(L_hat, dtype=np.float64)[:n, :n])
    check_finite(L_hat, 'potrf factor (lower triangle)')
    if L_ref is None:
        L_ref = scipy.linalg.cholesky(A, lower=True, check_finite=False)
    be_ref = cholesky_backward_error(A, L_ref)
    be = cholesky_backward_error(A, L_hat)
    limit = max(8 * be_ref, 64 * n * U)
    if not be <= limit:
        raise AssertionError('potrf: backward error %.3e > %.3e (LAPACK: %.3e)' % (be, limit, be_ref))
    if forward_tol is not None:
        err = np.max(np.abs(L_hat - np.tril(L_ref))) / np.max(np.abs(L_ref))
        if not err <= forward_tol:
            raise AssertionError('potrf: %.3e from LAPACK\'s factor (> %.1e)' % (err, forward_tol))
