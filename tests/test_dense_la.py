"""The dense-solve and Nystroem building blocks of the C ABI (csrc/solve.cu, csrc/nystroem.cu) against FP64
NumPy / LAPACK at the shapes the large-system solver runs, at block (NB = 128, NBO = 256 / 512 / 1024), tile
(128 x 128, 1024-row super-tiles) and chunk (256 rows) edges, with padded row strides.

Canaries: every padding column (ld > width), every row past the end of an output and every strictly upper
triangle a routine must not use holds NaN on input.  Results must be free of NaN where they are defined, and
padding columns of outputs must be bit-identical to what was there before the call.  The error bounds are the
ones of tests/la_checks.py."""

import functools

import numpy as np
import pytest

import la_checks as lc

pytestmark = pytest.mark.gpu

NAN = np.nan


@pytest.fixture(scope='module')
def lib():
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return _lib.lib()


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _host(t):
    import torch

    torch.cuda.synchronize()
    return t.cpu().numpy()


def _stream():
    from sgdml_b200 import _lib

    return _lib.current_stream()


def _check(rc, what):
    from sgdml_b200 import _lib

    _lib.check(rc, what)


def _even_pad(m):
    """The smallest even row stride with at least one padding column."""
    return m + 1 if m % 2 else m + 2


@functools.lru_cache(maxsize=None)
def _spd(n, rank=None, seed=0):
    """Symmetric positive definite, condition number below ~100: G G^T / r + I with G (n x r)."""
    r = n if rank is None else min(rank, n)
    G = np.random.default_rng(1000 + n + seed).standard_normal((n, r))
    A = G @ G.T / r
    A[np.diag_indices(n)] += 1.0
    return A


@functools.lru_cache(maxsize=None)
def _chol(n, rank=None):
    import scipy.linalg

    return scipy.linalg.cholesky(_spd(n, rank), lower=True, check_finite=False)


def _bits_equal(a, b):
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


# ================================================================================================ trsm_right_lt
@pytest.mark.parametrize('ldx_kind', ['tight', 'even', 'plus7'])
@pytest.mark.parametrize('n_rows', [1, 63, 64, 65, 4097])
@pytest.mark.parametrize('m', [1, 127, 128, 129, 351, 1107])
def test_trsm_right_lt(lib, m, n_rows, ldx_kind):
    """X <- X L^-T: one substitution strip per 128 columns plus the DMMA update of the later column blocks
    (m > 128), 64-row strips (n_rows at the strip edges)."""
    L = _chol(m)
    ldl = _even_pad(m)
    ldx = {'tight': m, 'even': _even_pad(m), 'plus7': m + 7}[ldx_kind]
    X0 = np.random.default_rng(7 * m + n_rows).standard_normal((n_rows, m))
    Lh = lc.nan_upper(L, ldl)
    Xh = lc.with_padding(X0, ldx)
    Ld, Xd = _dev(Lh), _dev(Xh)
    _check(lib.sgdml_b200_trsm_right_lt(Ld.data_ptr(), m, ldl, Xd.data_ptr(), n_rows, ldx, _stream()), 'trsm_right_lt')
    out = _host(Xd)
    assert _bits_equal(_host(Ld), Lh)  # L is an input only
    lc.check_padding_unchanged(Xh, out, m, 'X')
    lc.check_trsm_right_lt(L, X0, out, cond_ok=True)


# ================================================================================================ gram_tn
@pytest.mark.parametrize('m', [1, 108, 129, 1025, 2100])
@pytest.mark.parametrize('n_rows', [1, 33, 1081, 20000])
def test_gram_tn(lib, n_rows, m):
    """C = X^T X + lam I (lower triangle): odd n_rows takes the zero-padded transpose, m > 1024 several
    super-tile rows of the triangular raster."""
    X = np.random.default_rng(n_rows + 3 * m).standard_normal((n_rows, m))
    lam = 0.37
    ldx, ldc = m + 1, _even_pad(m)
    Xh = lc.with_padding(X, ldx)
    Ch = np.full((m, ldc), NAN)
    Xd, Cd = _dev(Xh), _dev(Ch)
    _check(lib.sgdml_b200_gram_tn(Xd.data_ptr(), n_rows, m, ldx, lam, Cd.data_ptr(), ldc, _stream()), 'gram_tn')
    C = _host(Cd)
    assert _bits_equal(_host(Xd), Xh)
    lc.check_padding_unchanged(Ch, C, m, 'C')
    lc.check_gram(X, C, lam)


# ================================================================================================ row_sqnorms
@pytest.mark.parametrize('out_on', ['host', 'device'])
@pytest.mark.parametrize('m', [1, 31, 32, 33, 1025])
def test_row_sqnorms(lib, m, out_on):
    n_rows = 777
    X = np.random.default_rng(m).standard_normal((n_rows, m))
    Xd = _dev(lc.with_padding(X, m + 1))
    out = np.full(n_rows + 1, NAN)  # one canary past the end
    od = out if out_on == 'host' else _dev(out)
    from sgdml_b200 import _lib

    _check(lib.sgdml_b200_row_sqnorms(Xd.data_ptr(), n_rows, m, m + 1, _lib.ptr(od), _stream()), 'row_sqnorms')
    res = out if out_on == 'host' else _host(od)
    assert np.isnan(res[-1]) and _bits_equal(res[-1:], np.full(1, NAN))
    lc.check_row_sqnorms(X, res[:n_rows])


# ================================================================================================ Nystroem products
@pytest.mark.parametrize('m', [1, 97, 128, 129, 1000])
@pytest.mark.parametrize('n_rows', [1, 255, 256, 257, 100003])
def test_nystroem_apply_project_expand(lib, n_rows, m):
    """P v = (X (X^T v) - v)/lam and its two halves, vectors on the host and on the device.  n_rows at the edges
    of the 256-row chunks of X^T v.  Deterministic: repeated calls, host and device vectors, and apply against
    project + expand are bit-identical, which the row-sharded CG relies on (every rank must compute the same
    scalars)."""
    from sgdml_b200 import _lib

    rng = np.random.default_rng(n_rows + m)
    X = rng.standard_normal((n_rows, m)) / np.sqrt(m)
    v = rng.standard_normal(n_rows)
    lam = 1e-2
    ldx = m + 1
    Xd = _dev(lc.with_padding(X, ldx))
    del rng
    results = {}
    for place in ('host', 'device'):
        def buf(k):
            a = np.full(k + 1, NAN)  # one canary past the end
            return a if place == 'host' else _dev(a)

        def get(b):
            return b if place == 'host' else _host(b)

        vv = v.copy() if place == 'host' else _dev(v)
        out_a, out_a2, t, out_e = buf(n_rows), buf(n_rows), buf(m), buf(n_rows)
        for o in (out_a, out_a2):
            _check(lib.sgdml_b200_nystroem_apply(Xd.data_ptr(), n_rows, m, ldx, lam, _lib.ptr(vv), _lib.ptr(o), _stream()), 'apply')
        _check(lib.sgdml_b200_nystroem_project(Xd.data_ptr(), n_rows, m, ldx, _lib.ptr(vv), _lib.ptr(t), _stream()), 'project')
        _check(
            lib.sgdml_b200_nystroem_expand(Xd.data_ptr(), n_rows, m, ldx, lam, _lib.ptr(t), _lib.ptr(vv), _lib.ptr(out_e), _stream()),
            'expand',
        )
        res = [get(b) for b in (out_a, out_a2, t, out_e)]
        for r in res:
            assert np.isnan(r[-1]) and _bits_equal(r[-1:], np.full(1, NAN))  # nothing written past the end
        results[place] = [r[:-1] for r in res]
    a, a2, t, e = results['host']
    assert _bits_equal(a, a2)
    assert _bits_equal(a, e)
    for x, y in zip(results['host'], results['device']):
        assert _bits_equal(x, y)
    lc.check_project(X, v, t)
    lc.check_expand(X, t, v, lam, e)
    lc.check_apply(X, v, lam, a)


# ================================================================================================ gather_rows_neg / add_diag
@pytest.mark.parametrize('idx_on', ['host', 'device'])
@pytest.mark.parametrize('m', [1, 129, 2000])
def test_gather_rows_neg_and_add_diag(lib, m, idx_on):
    """K_mm = -X[rows, :] with unsorted, repeated row indices, then the diagonal shift: both exact."""
    import torch

    rng = np.random.default_rng(m)
    n_rows = 2 * m + 5
    ldx, ldo = m + 3, m + 1
    X = rng.standard_normal((n_rows, m))
    idx = rng.integers(0, n_rows, size=m).astype(np.int64)
    if m > 1:
        idx[-1] = idx[0]  # a repeated index
        idx[:2] = [n_rows - 1, 0]  # unsorted, both ends
    Xh = lc.with_padding(X, ldx)
    Oh = np.full((m, ldo), NAN)
    Xd, Od = _dev(Xh), _dev(Oh)
    idx_arg = idx if idx_on == 'host' else torch.from_numpy(idx).cuda()
    from sgdml_b200 import _lib

    _check(lib.sgdml_b200_gather_rows_neg(Xd.data_ptr(), ldx, m, _lib.ptr(idx_arg), Od.data_ptr(), ldo, _stream()), 'gather')
    O = _host(Od)
    assert np.array_equal(O[:, :m], -X[idx])
    lc.check_padding_unchanged(Oh, O, m, 'out')
    assert _bits_equal(_host(Xd), Xh)
    _check(lib.sgdml_b200_add_diag(Od.data_ptr(), m, ldo, 0.375, _stream()), 'add_diag')
    expect = O.copy()
    expect[np.diag_indices(m)] += 0.375
    assert _bits_equal(_host(Od), expect)


# ================================================================================================ potrf
POTRF_N = [1, 127, 129, 255, 257, 4095, 4097]


def _potrf_inputs(n, lda):
    """A in a (n x lda) buffer with NaN in the strictly upper triangle and the padding column; and the same A
    with its full symmetric storage and no canaries."""
    A = _spd(n, rank=256)
    return A, lc.nan_upper(np.tril(A), lda), lc.with_padding(A, lda, 0.0)


@pytest.mark.parametrize('slices', [0, 7])
@pytest.mark.parametrize('pad', [0, 1])
@pytest.mark.parametrize('n', POTRF_N)
def test_potrf(lib, n, pad, slices, monkeypatch):
    """Cholesky at the inner (NB = 128) and outer block edges (NBO = 256 below n = 4096, 512 from there:
    4097 is one column past the outer blocks), lda = n and the padded lda = n + 1 of the analytic solver and the
    Nystroem squares, FP64 and int8-slice trailing updates.  The upper triangle is never read (NaN there changes
    no bit of L) and the padding column is never written."""
    monkeypatch.setenv('SGDML_B200_OZAKI_SLICES', str(slices))
    lda = n + pad
    A, Ac, Afull = _potrf_inputs(n, lda)
    Ad, Ad2 = _dev(Ac), _dev(Afull)
    for buf in (Ad, Ad2):
        _check(lib.sgdml_b200_potrf(buf.data_ptr(), n, lda, _stream()), 'potrf')
    out, out2 = _host(Ad), _host(Ad2)
    lc.check_padding_unchanged(Ac, out, n, 'A')
    lc.check_padding_unchanged(Afull, out2, n, 'A')
    low = np.tril_indices(n)
    assert _bits_equal(out[:, :n][low], out2[:, :n][low])  # the upper triangle is not read
    lc.check_cholesky(A, out[:, :n], L_ref=_chol(n, 256), forward_tol=1e-12)
    if n == 129:  # host buffer: staged through the device, same bits
        h = Ac.copy()
        _check(lib.sgdml_b200_potrf(h.ctypes.data, n, lda, None), 'potrf')
        lc.check_padding_unchanged(Ac, h, n, 'A (host)')
        assert _bits_equal(h[:, :n][low], out[:, :n][low])


def test_potrf_sgdml_system(lib):
    """The matrix the analytic solver factorises, -K + lam I of a golden task (condition ~1e11), assembled by the
    engine into a padded buffer (odd n + 1 row stride): backward error against LAPACK's on the same matrix."""
    from conftest import load_golden
    from sgdml_b200 import _lib

    g = load_golden('n9_m16_s6')
    N, M = int(g['n_atoms']), g['R_desc'].shape[0]
    n = 3 * N * M
    lin = np.ascontiguousarray(g['tril_perms_lin'], dtype=np.int64)
    S = len(lin) // g['R_desc'].shape[1]
    ldk = n + 1
    Kh = np.full((n, ldk), NAN)
    Kd = _dev(Kh)
    _check(
        lib.sgdml_b200_assemble(
            _lib.ptr(np.ascontiguousarray(g['R_desc'])), _lib.ptr(np.ascontiguousarray(g['R_d_desc'])), _lib.ptr(lin),
            N, M, S, float(g['sig']), None, n, -1.0, Kd.data_ptr(), ldk, _stream(),
        ),
        'assemble',
    )
    _check(lib.sgdml_b200_add_diag(Kd.data_ptr(), n, ldk, float(g['lam']), _stream()), 'add_diag')
    A = _host(Kd)[:, :n].copy()
    assert np.max(np.abs(A + g['K'] - float(g['lam']) * np.eye(n))) < 1e-11 * np.max(np.abs(g['K']))
    Kd[:, :n] = Kd[:, :n].tril() + Kd.new_full((n, n), NAN).triu(1)
    Kc = _host(Kd)
    _check(lib.sgdml_b200_potrf(Kd.data_ptr(), n, ldk, _stream()), 'potrf')
    out = _host(Kd)
    lc.check_padding_unchanged(Kc, out, n, 'K')
    lc.check_cholesky(A, out[:, :n])


# ------------------------------------------------------------------------------------------------ potrf failures
FAIL_N = 4100


@functools.lru_cache(maxsize=1)
def _fail_base():
    return _spd(FAIL_N, rank=64)


def _not_pd_at(minor):
    """A whose leading minors of order < `minor` are positive definite and whose pivot `minor` is -1."""
    import scipy.linalg

    A = _fail_base().copy()
    k = minor - 1
    if k == 0:
        A[0, 0] = -1.0
        return A
    Lk = scipy.linalg.cholesky(A[:k, :k], lower=True, check_finite=False)
    l = scipy.linalg.solve_triangular(Lk, A[:k, k], lower=True, check_finite=False)
    A[k, k] = l @ l - 1.0  # Schur complement -1
    return A


@pytest.mark.parametrize('slices', [0, 7])
@pytest.mark.parametrize('minor', [1, 128, 129, 513, 700, 'nan'])
def test_potrf_reports_failing_minor(lib, minor, slices, monkeypatch):
    """info = the order of the first leading minor that is not positive definite: at the first column, the last
    and first columns of an inner block, the first column of an outer block (NBO = 512), and 700, inside the
    second outer block, after a lazy trailing update; and a NaN on the diagonal (at 301)."""
    from sgdml_b200 import _lib

    monkeypatch.setenv('SGDML_B200_OZAKI_SLICES', str(slices))
    if minor == 'nan':
        A = _fail_base().copy()
        A[300, 300] = NAN
        expect = 301
    else:
        A, expect = _not_pd_at(minor), minor
    Ad = _dev(lc.nan_upper(np.tril(A), FAIL_N + 1))
    rc = lib.sgdml_b200_potrf(Ad.data_ptr(), FAIL_N, FAIL_N + 1, _stream())
    assert rc == expect
    with pytest.raises(np.linalg.LinAlgError, match='%d-th leading minor' % expect):
        _lib.check(rc, 'potrf')


# ================================================================================================ potrs
@pytest.mark.parametrize('nrhs', [1, 2, 129, 300])
@pytest.mark.parametrize('n', [1, 127, 129, 1000])
def test_potrs(lib, n, nrhs):
    """L L^T X = B with L from LAPACK (NaN in its upper triangle and padding column), B with padding columns
    (ldb = nrhs + 3)."""
    A = _spd(n)
    L = _chol(n)
    lda, ldb = n + 1, nrhs + 3
    B = np.random.default_rng(n * nrhs).standard_normal((n, nrhs))
    Lh, Bh = lc.nan_upper(L, lda), lc.with_padding(B, ldb)
    Ld, Bd = _dev(Lh), _dev(Bh)
    _check(lib.sgdml_b200_potrs(Ld.data_ptr(), n, lda, Bd.data_ptr(), nrhs, ldb, _stream()), 'potrs')
    X = _host(Bd)
    assert _bits_equal(_host(Ld), Lh)
    lc.check_padding_unchanged(Bh, X, nrhs, 'B')
    lc.check_potrs(A, L, B, X, cond_ok=True)
    if n == 129:  # host buffers: staged, same bits
        Xh = Bh.copy()
        _check(lib.sgdml_b200_potrs(Lh.ctypes.data, n, lda, Xh.ctypes.data, nrhs, ldb, None), 'potrs')
        assert _bits_equal(Xh, X)
