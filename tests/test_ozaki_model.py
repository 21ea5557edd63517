"""CPU checks of the exact model of the int8-slice GEMM (tests/ozaki_model.py): its error against the exact product
stays within the componentwise bound `method_bound` for every slice count, and the bit-for-bit comparison the GPU
tests make with it rejects synthetic defects that the former tolerance check (1e-12 of |A||B|^T) accepts."""

import numpy as np
import pytest

import ozaki_model as om

SLICES = [2, 3, 4, 5, 6, 7]


def _exact_dots(A, B):
    """A B^T exactly: every double is an integer multiple of 2^-1074, so the scaled entries are Python integers and
    their products and sums are exact.  Returns (integer matrix, power of two it is scaled by)."""
    def one(x):
        num, den = x.as_integer_ratio()  # den is a power of two <= 2^1074
        return num * (2**1074 // den)

    def ints(X):
        return np.array([[one(x) for x in row] for row in X.tolist()], dtype=object)

    return ints(A) @ ints(B).T, 2 * 1074


def _data(kind, m, n, k, seed):
    rng = np.random.default_rng([m, n, k, seed])
    if kind == 'normal':
        return rng.standard_normal((m, k)), rng.standard_normal((n, k))
    if kind == 'rows_2^20':
        return (np.ldexp(rng.standard_normal((m, k)), rng.integers(-20, 21, size=(m, 1))),
                np.ldexp(rng.standard_normal((n, k)), rng.integers(-20, 21, size=(n, 1))))
    if kind == 'sparse':  # zero rows, single nonzeros, a row maximum far above the rest
        A, B = rng.standard_normal((m, k)), rng.standard_normal((n, k))
        A[0] = 0.0
        A[1] = 0.0
        A[1, k // 2] = -3.0
        B[0, 0] = 2.0**30
        B[1] = np.ldexp(B[1], -40)
        return A, B
    if kind == 'extreme_slices':  # every entry just below the row maximum: first slices of 64
        A = np.where(rng.random((m, k)) < 0.5, -1.0, 1.0) * (1 - 2.0**-53)
        B = np.where(rng.random((n, k)) < 0.5, -1.0, 1.0) * (1 - rng.random((n, k)) * 2.0**-20)
        return A, B
    if kind == 'ties':  # entries on the half-way grid 2^-(7p + 1) of the slicing: rint's ties
        p = rng.integers(1, 7, size=(m, k))
        A = rng.integers(-60, 61, size=(m, k)) / 128.0 + np.where(rng.random((m, k)) < 0.5, -1, 1) * 2.0 ** (-7 * p - 1)
        A[:, 0] = 0.45
        return A, rng.standard_normal((n, k))
    raise ValueError(kind)


KINDS = ['normal', 'rows_2^20', 'sparse', 'extreme_slices', 'ties']


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('k', [1, 37, 300])
def test_model_within_method_bound(k, kind):
    """|U - alpha A B^T| <= method_bound entry by entry, for S = 2..7 and alpha in {1, -0.3}, against the exact product."""
    m, n = 9, 7
    A, B = _data(kind, m, n, k, 0)
    P, sh = _exact_dots(A, B)
    ea, _ = om.row_exponents(A)
    eb, _ = om.row_exponents(B)
    from fractions import Fraction

    for S in SLICES:
        for alpha in (1.0, -0.3):
            U = om.gemm(A, B, np.zeros((m, n)), alpha, S, overwrite=True)
            bnd = om.method_bound(ea, eb, k, S, alpha)
            fa = Fraction(alpha)
            for i in range(m):
                for j in range(n):
                    err = abs(Fraction(float(U[i, j])) - fa * Fraction(P[i, j], 2**sh))
                    assert err <= Fraction(float(bnd[i, j])), (S, alpha, i, j, float(err), float(bnd[i, j]))


def test_level_sums_fit_int32():
    """At k = 16384 the level sums of the largest slices stay below 2^31 (the kernel's int32 accumulators), as the
    bound 64^2 k S < 2^31 says."""
    S = 7
    assert 64 * 64 * om.K_MAX * S < 2**31
    A, B = _data('extreme_slices', 2, 2, om.K_MAX, 1)
    _, sa, _ = om.split(A, S)
    _, sb, _ = om.split(B, S)
    assert np.max(np.abs(sa)) == 64
    for lev in om.levels(sa, sb, S):
        assert np.max(np.abs(lev)) < 2**31


def test_tri_write_set():
    """tri: whole 128 x 32 tiles that reach the lower triangle, the entries above the diagonal inside them included."""
    mask = om.tri_mask(300, 300)
    assert mask[np.tril_indices(300)].all()
    assert mask[0, 127] and not mask[0, 128] and mask[127, 127] and not mask[127, 128] and mask[128, 255]
    assert not mask[128, 256] and mask[299, 299]


def _case(m, n, k, seed=0):
    rng = np.random.default_rng([m, n, k, seed])
    A = np.ldexp(rng.standard_normal((m, k)), rng.integers(-3, 4, size=(m, 1)))
    return A, rng.standard_normal((n, k)), rng.standard_normal((m, n))


@pytest.mark.parametrize('S', [2, 5, 7])
@pytest.mark.parametrize('defect', om.DEFECTS)
@pytest.mark.parametrize('shape', [(128, 64, 128), (300, 200, 130), (129, 65, 1000)], ids=lambda s: '%dx%dx%d' % s)
def test_exact_comparison_rejects_defect(shape, defect, S):
    """Each synthetic defect changes the bits of C somewhere, so the GPU tests' `==` comparison fails on it."""
    A, B, C0 = _case(*shape)
    overwrite = defect == 'ignore_overwrite'
    good = om.gemm(A, B, C0, 1.0, S, overwrite=overwrite)
    bad = om.gemm(A, B, C0, 1.0, S, overwrite=overwrite, defect=defect)
    diff = good.view(np.int64) != bad.view(np.int64)
    assert diff.any()
    if defect in ('drop_pair', 'level_weight'):
        i, j = np.argwhere(diff)[0]
        why = om.explain(A, B, 1.0, S, bad[i, j] - C0[i, j], good[i, j] - C0[i, j], i, j)
        assert ('pair (%d, 1)' % S if defect == 'drop_pair' else 'level') in why, why


@pytest.mark.parametrize('shape', [(128, 64, 128), (300, 200, 130), (129, 65, 1000)], ids=lambda s: '%dx%dx%d' % s)
def test_former_tolerance_accepts_dropped_pair(shape):
    """Why the GPU tests compare bits: a kernel that skipped the slice pair (7, 1) passes the former check
    max |C - C_ref| / (|A| |B|^T) < 1e-12 at the former tests' shapes, while thousands of entries differ from the exact
    model."""
    rng = np.random.default_rng(0)
    m, n, k = shape
    A, B, C0 = rng.standard_normal((m, k)), rng.standard_normal((n, k)), rng.standard_normal((m, n))
    bad = om.gemm(A, B, C0, 1.0, 7, defect='drop_pair')
    assert np.max(np.abs(bad - (C0 + A @ B.T)) / (np.abs(A) @ np.abs(B).T)) < 1e-12
    assert np.count_nonzero(bad != om.gemm(A, B, C0, 1.0, 7)) > 1000


def test_non_finite_rows_give_nan_rows_and_columns():
    A, B, C0 = _case(40, 35, 20)
    A[3, 7], B[5, 0], B[9, 19] = np.nan, np.inf, -np.inf
    C = om.gemm(A, B, C0, -1.0, 6)
    nan = np.zeros(C.shape, dtype=bool)
    nan[3, :] = nan[:, 5] = nan[:, 9] = True
    assert np.array_equal(np.isnan(C), nan)


def test_update_equals_two_step_scaling_in_the_normal_range():
    """ldexp(fl(alpha V), ea + eb) is the former epilogue's (V alpha 2^ea) 2^eb wherever neither factor over- or
    underflows, so finite normal-range outputs keep their bits under the combined scaling."""
    A, B, C0 = _case(130, 70, 200)
    A = np.ldexp(A, np.random.default_rng(1).integers(-40, 41, size=(130, 1)))
    for S, alpha in ((7, 1.0), (5, -1.0), (4, 0.3)):
        ea, sa, _ = om.split(A, S)
        eb, sb, _ = om.split(B, S)
        V = om.combine(om.levels(sa, sb, S), S)
        two_step = V * (alpha * np.ldexp(1.0, ea))[:, None] * np.ldexp(1.0, eb)[None, :]
        assert np.array_equal(om.scale(V, alpha, ea, eb, np.zeros(130, bool), np.zeros(70, bool)), two_step)
