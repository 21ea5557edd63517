"""The FP64 GEMM of csrc/solve.cu (launch_gemm: k_gemm_nt_tma, k_gemm_nt, k_gemm_nt_naive) in every mode,
rasterisation and call shape its callers issue, through the test hook sgdml_b200_gemm_nt_args.

Two kinds of operands.  'int': small integers (|a|, |b| <= 7, |c0| <= 1000), for which every partial sum is exact in
FP64 in any order, compared with `==` against the product NumPy forms on the host (exact for the same reason): a
dropped, duplicated or misrouted element shows, and the failure names the 128 x 128 tiles.  'scaled': standard-normal
operands whose rows are scaled by 2^e, e in [-20, 20], checked with the componentwise bound of
la_checks.check_gemm_nt, which a small row cannot hide in.

Canaries.  Every operand and every C is a window of a NaN-filled device buffer with padding columns, one more row
after the last, and, where the caller passes a window of a wider matrix, that matrix around it.  No NaN may reach the
result, and everything outside the result must be bit-identical after the call.

The result of a call with tri = 1 (m == n) is the lower triangle, col <= row.  The tile kernels compute whole tiles:
they also write the entries above the diagonal inside the diagonal tiles (from whatever those held), and leave every
tile (ti, tj) with tj > ti untouched.  The scalar kernel writes no entry with col > row.  The tests put NaN in the
whole strictly upper triangle of C and assert exactly that.

Kernels: 'tma' (variant 3, the default), 'cpasync' (variant 0), 'scalar' (variant 2; also what operands that the tile
kernels cannot load are routed to)."""

import functools

import numpy as np
import pytest

import la_checks as lc

pytestmark = pytest.mark.gpu

NAN = float('nan')
T = lc.GEMM_TILE
KERNELS = {'cpasync': 0, 'scalar': 2, 'tma': 3}
TILE_KERNELS = ['cpasync', 'tma']
ALL_KERNELS = ['cpasync', 'tma', 'scalar']


@pytest.fixture(scope='module')
def lib():
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return _lib.lib()


def _check(rc, what):
    from sgdml_b200 import _lib

    _lib.check(rc, what)


def _stream():
    from sgdml_b200 import _lib

    return _lib.current_stream()


def _up(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _bits(t):
    import torch

    return t.view(torch.int64)


def _even(x):
    return x + x % 2


class Buf:
    """A (rows x ld) row-major device matrix that starts `off` doubles into its allocation.  Its first `cols`
    columns (all of them by default) hold NaN until a test fills a window, and are the part compared before and
    after a call.  `storage`: an existing flat tensor to live in (the strided 20 GB cases, where only the leading
    columns are ever touched)."""

    def __init__(self, rows, ld, off=0, cols=None, storage=None):
        import torch

        self.rows, self.ld, self.cols = rows, ld, ld if cols is None else cols
        flat = storage if storage is not None else torch.empty(off + rows * ld, dtype=torch.float64, device='cuda')
        assert flat.numel() >= off + rows * ld
        self.flat = flat
        self.mat = flat[off : off + rows * ld].view(rows, ld)
        self.mat[:, : self.cols] = NAN

    def ptr(self, r=0, c=0):
        assert 0 <= r < self.rows and 0 <= c < self.ld
        return self.mat[r:, c:].data_ptr()

    def snapshot(self):
        return self.mat[:, : self.cols].clone()

    def changed(self, snap):
        return _bits(self.mat[:, : self.cols]) != _bits(snap)


def _assert_unchanged(buf, snap, what, window=None, may_write=None):
    """Every entry of buf is bit-identical to snap, except, inside window = (r0, c0, m, n), those that may_write (a
    bool m x n mask; None = the whole window) allows."""
    changed = buf.changed(snap)
    if window is not None:
        r0, c0, m, n = window
        sub = changed[r0 : r0 + m, c0 : c0 + n]
        if may_write is None:
            sub.fill_(False)
        else:
            sub.logical_and_(~may_write)
    if bool(changed.any()):
        r, c = changed.nonzero()[0].tolist()
        rel = ' = (%d, %d) of the result window, tile (%d, %d)' % (r - r0, c - c0, (r - r0) // T, (c - c0) // T) if window else ''
        raise AssertionError('%s: %d entries outside the result were written; first at (%d, %d) of the buffer%s'
                             % (what, int(changed.sum()), r, c, rel))


def _may_write(kernel, m, n):
    """What a tri = 1 call may write: col <= row for the scalar kernel, the tiles tj <= ti for the tile kernels."""
    import torch

    r = torch.arange(m, device='cuda')[:, None]
    c = torch.arange(n, device='cuda')[None, :]
    return (c <= r) if kernel == 'scalar' else (c // T <= r // T)


def _call(lib, kernel, m, n, k, A, lda, B, ldb, C, ldc, alpha=1.0, beta=1.0, mode=0, tri=0, flag=None):
    import torch

    _check(lib.sgdml_b200_set_gemm_variant(KERNELS[kernel]), 'set_gemm_variant')
    try:
        rc = lib.sgdml_b200_gemm_nt_args(m, n, k, alpha, A, lda, B, ldb, beta, C, ldc, mode, tri, flag, _stream())
        _check(rc, 'gemm_nt_args')
        torch.cuda.synchronize()
    finally:
        lib.sgdml_b200_set_gemm_variant(3)


@functools.lru_cache(maxsize=2)
def _case_data(m, n, k, data, same_ab, seed=0):
    """Host operands A (m x k), B (n x k), C0 (m x n) and, for 'int', the exact product A B^T."""
    rng = np.random.default_rng([m, n, k, seed])
    if data == 'int':
        A = rng.integers(-7, 8, size=(m, k)).astype(np.float64)
        B = A if same_ab else rng.integers(-7, 8, size=(n, k)).astype(np.float64)
        C0 = rng.integers(-1000, 1001, size=(m, n)).astype(np.float64)
        P = A @ B.T
        assert np.array_equal(P, P.astype(np.int64)) and np.max(np.abs(P)) <= 49 * k
        return A, B, C0, P
    ea = rng.integers(-20, 21, size=m)
    A = np.ldexp(rng.standard_normal((m, k)), ea[:, None])
    eb = ea if same_ab else rng.integers(-20, 21, size=n)
    B = A if same_ab else np.ldexp(rng.standard_normal((n, k)), eb[:, None])
    C0 = np.ldexp(rng.standard_normal((m, n)) * np.sqrt(k), ea[:, None] + eb[None, :])
    return A, B, C0, None


def _run(lib, kernel, data, s, C0=None):
    """One call as the dict s describes it: m, n, k, mode, tri, alpha, beta and A, B, C = (Buf, first row, first
    column).  Fills the windows (C0 given: C already holds it), calls, asserts that nothing outside the result
    changed, verifies the result and returns it."""
    import torch

    m, n, k, mode, tri = s['m'], s['n'], s['k'], s['mode'], s.get('tri', 0)
    alpha, beta = s.get('alpha', 1.0), s.get('beta', 1.0)
    same_ab = s['A'] == s['B']
    hA, hB, hC0, P = _case_data(m, n, k, data, same_ab, s.get('seed', 0))
    (Ab, ar, ac), (Bb, br, bc), (Cb, cr, cc) = s['A'], s['B'], s['C']
    Ab.mat[ar : ar + m, ac : ac + k] = _up(hA)
    if not same_ab:
        Bb.mat[br : br + n, bc : bc + k] = _up(hB)
    reads_c = mode == 1 or beta != 0.0
    if C0 is not None:
        hC0 = C0
    elif reads_c:  # otherwise C keeps its NaN: it must not be read
        c = _up(hC0)
        if tri:
            c = torch.where(torch.ones(m, n, dtype=torch.bool, device='cuda').tril(), c, NAN)
        Cb.mat[cr : cr + m, cc : cc + n] = c
    bufs = {id(b): b for b in (Ab, Bb, Cb)}
    snaps = {i: b.snapshot() for i, b in bufs.items()}
    _call(lib, kernel, m, n, k, Ab.ptr(ar, ac), Ab.ld, Bb.ptr(br, bc), Bb.ld, Cb.ptr(cr, cc), Cb.ld, alpha, beta, mode,
          tri)
    what = '%s %dx%dx%d mode %d tri %d' % (kernel, m, n, k, mode, tri)
    for i, b in bufs.items():
        if b is Cb:
            _assert_unchanged(b, snaps[i], what, (cr, cc, m, n), _may_write(kernel, m, n) if tri else None)
        else:
            _assert_unchanged(b, snaps[i], what + ' (operand buffer)')
    del snaps
    got = Cb.mat[cr : cr + m, cc : cc + n].cpu().numpy()
    if mode == 1:  # accumulators start from C: alpha and beta are not used
        alpha = beta = 1.0
    if data == 'int':
        assert alpha == 1.0 and beta in (0.0, 1.0)
        ref = P + hC0 if reads_c else P
        bad = ~(got == ref)  # NaN differs
        if tri:
            bad &= np.tri(m, n, dtype=bool)
        if bad.any():
            r, c = np.argwhere(bad)[0]
            raise AssertionError('%s: %d entries differ from the exact product, in tiles %s; first at (%d, %d): %r, expected %r'
                                 % (what, int(bad.sum()), lc.tiles_of(bad), r, c, float(got[r, c]), float(ref[r, c])))
    else:
        lc.check_gemm_nt(hA, hB, hC0 if reads_c else None, got, alpha, beta, bool(tri), what)
    return got


def test_hook_rejects_what_it_cannot_launch(lib):
    """mode and tri outside {0, 1}, tri on a non-square C, strides shorter than a row and host pointers are argument
    errors, reported before anything is launched: C keeps its bits."""
    import torch

    A, B, C = Buf(9, 8), Buf(9, 8), Buf(9, 8)
    A.mat[:], B.mat[:], C.mat[:] = 1.0, 1.0, 3.0
    snap = C.snapshot()
    host = np.ones((9, 8))
    ok = dict(m=8, n=8, k=8, A=A.ptr(), lda=8, B=B.ptr(), ldb=8, C=C.ptr(), ldc=8, mode=0, tri=0, flag=None)
    bad = [dict(mode=2), dict(mode=-1), dict(tri=2), dict(tri=1, m=6), dict(lda=6), dict(ldb=6), dict(ldc=6), dict(k=0),
           dict(A=host.ctypes.data), dict(B=host.ctypes.data), dict(C=host.ctypes.data), dict(flag=host.ctypes.data), dict(A=None)]
    for change in bad:
        a = dict(ok, **change)
        rc = lib.sgdml_b200_gemm_nt_args(a['m'], a['n'], a['k'], 1.0, a['A'], a['lda'], a['B'], a['ldb'], 1.0, a['C'], a['ldc'],
                                         a['mode'], a['tri'], a['flag'], _stream())
        assert rc == -1000, change  # SGDML_B200_ERR_ARG
    torch.cuda.synchronize()
    _assert_unchanged(C, snap, 'rejected calls')


# ================================================================================================ (a), (b) the edge grid
MN = [1, 2, 127, 128, 129, 255, 257, 1025]  # tile edges; an odd n takes the single-column tail store
# KT = 1 ... 5 k-tiles of 32 around the 3-stage ring, the k tail inside the first and inside the second 16-column
# box of a stage, and a second box that is entirely out of bounds (k = 2, 14, 16 mod 32)
KS = [2, 14, 16, 18, 30, 32, 34, 62, 64, 66, 94, 96, 98, 128, 130, 1024, 1026]
GRID = sorted(
    {(MN[i % 8], MN[(3 * i + 5) % 8], k) for i, k in enumerate(KS)}
    | {(MN[(3 * i + 1) % 8], MN[(i + i // 8 + 2) % 8], k) for i, k in enumerate(KS)}
    | {(1025, 1025, 1026), (257, 257, 34)}
)
GRID_SMALL = [c for c in GRID if max(c[0], c[1]) <= 257]
FORMS = {  # name -> (mode, alpha, beta)
    'mode0_beta0': (0, 1.0, 0.0),
    'mode0_beta1': (0, 1.0, 1.0),
    'mode0_general': (0, 0.75, -1.25),
    'mode1': (1, 1.0, 1.0),
}


def _shape_id(c):
    return '%dx%dx%d' % c


def _plain_case(m, n, k, form, tri=0, lda=None, ldb=None, ldc=None, off=(0, 0, 0)):
    """Three separate buffers with padding columns, a NaN row after the last, and optionally `off` doubles of
    misalignment each."""
    mode, alpha, beta = FORMS[form]
    lda = k + 2 if lda is None else lda
    ldb = k + 4 if ldb is None else ldb
    ldc = _even(n) + 2 if ldc is None else ldc
    A, B, C = Buf(m + 1, lda, off[0]), Buf(n + 1, ldb, off[1]), Buf(m + 1, ldc, off[2])
    return dict(m=m, n=n, k=k, mode=mode, alpha=alpha, beta=beta, tri=tri, A=(A, 0, 0), B=(B, 0, 0), C=(C, 0, 0))


def test_grid_covers_every_edge():
    """Every m, n and k of the edge lists is in the grid the tile kernels run, and the scalar kernel's part of it
    reaches every value up to 257."""
    assert {c[0] for c in GRID} == set(MN) and {c[1] for c in GRID} == set(MN) and {c[2] for c in GRID} == set(KS)
    small = set(MN) - {1025}
    assert {c[0] for c in GRID_SMALL} == small and {c[1] for c in GRID_SMALL} == small


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('form', ['mode0_beta0', 'mode0_beta1', 'mode1'])
@pytest.mark.parametrize('shape', GRID, ids=_shape_id)
def test_exact_tile_kernels(lib, shape, form, kernel):
    """Integer operands over the edge grid: the result equals the exact product, entry for entry."""
    _run(lib, kernel, 'int', _plain_case(*shape, form))


@pytest.mark.parametrize('form', ['mode0_beta0', 'mode0_beta1', 'mode1'])
@pytest.mark.parametrize('shape', GRID_SMALL, ids=_shape_id)
def test_exact_scalar_kernel(lib, shape, form):
    _run(lib, 'scalar', 'int', _plain_case(*shape, form))


UNALIGNED = {  # what the tile kernels cannot load: each runs the scalar kernel whatever variant is selected
    'odd_k7': dict(k=7),
    'odd_k33': dict(k=33),
    'odd_k129': dict(k=129),
    'odd_lda': dict(k=34, lda=37),
    'odd_ldb': dict(k=34, ldb=35),
    'odd_ldc': dict(k=34, ldc=131),
    'A_8_bytes_off': dict(k=34, off=(1, 0, 0)),
    'B_8_bytes_off': dict(k=34, off=(0, 1, 0)),
    'C_8_bytes_off': dict(k=34, off=(0, 0, 1)),
}


@pytest.mark.parametrize('kernel', ['tma', 'scalar'])
@pytest.mark.parametrize('form', ['mode0_beta0', 'mode0_beta1', 'mode1'])
@pytest.mark.parametrize('layout', sorted(UNALIGNED))
def test_exact_unaligned_operands(lib, layout, form, kernel):
    """Odd k, odd row strides and pointers 8 bytes off 16-byte alignment, with the default kernel selected (the
    launch routes them to the scalar kernel) and with the scalar kernel selected."""
    _run(lib, kernel, 'int', _plain_case(257, 129, form=form, **UNALIGNED[layout]))


ACCURACY_SHAPES = [(129, 257, 66), (1025, 127, 130), (255, 1025, 1026), (2, 129, 34), (257, 255, 14), (128, 128, 96)]


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('form', ['mode0_beta0', 'mode0_general', 'mode1'])
@pytest.mark.parametrize('shape', ACCURACY_SHAPES, ids=_shape_id)
def test_componentwise_accuracy_tile_kernels(lib, shape, form, kernel):
    """Row-scaled normal operands, general alpha and beta: every entry within the componentwise bound."""
    _run(lib, kernel, 'scaled', _plain_case(*shape, form))


@pytest.mark.parametrize('form', ['mode0_beta0', 'mode0_general', 'mode1'])
@pytest.mark.parametrize('shape', [c for c in ACCURACY_SHAPES if max(c[:2]) <= 257], ids=_shape_id)
def test_componentwise_accuracy_scalar_kernel(lib, shape, form):
    _run(lib, 'scalar', 'scaled', _plain_case(*shape, form))


@pytest.mark.parametrize('kernel', ALL_KERNELS)
@pytest.mark.parametrize('data', ['int', 'scaled'])
@pytest.mark.parametrize('form', ['mode0_beta0', 'mode0_beta1', 'mode1'])
@pytest.mark.parametrize('n', [1, 129, 257, 300])
def test_tri_small(lib, n, form, data, kernel):
    """tri = 1 with all three kernels: the lower triangle is right, tiles above the diagonal keep their NaN bit for
    bit, and the scalar kernel leaves every entry with col > row alone."""
    _run(lib, kernel, data, _plain_case(n, n, 34, form, tri=1))


# ================================================================================================ (c) the callers' call shapes
def _potrf_inner(nbo, j, rem, pad):
    """potrf_device, inner update after panel j of the second outer block (K0 = NBO): C += (-X) X^T with
    A = the 128-column window at column 128 j of the (n x NBO) workspace W, B = the panel rows below the diagonal
    block and C = the columns of the outer block still to be factorised, both windows of the same rows of the
    (n x lda) matrix.  m = rem rows, n = min(NBO - 128 (j + 1), rem) columns (the outer block ends with the matrix)."""
    K0 = nbo
    k0 = K0 + 128 * j
    n_mat = k0 + 128 + rem
    K1 = min(K0 + nbo, n_mat)
    lda = _even(n_mat) + pad
    W, M = Buf(n_mat + 1, nbo), Buf(n_mat + 1, lda)
    return dict(m=rem, n=K1 - (k0 + 128), k=128, mode=1, tri=0, A=(W, k0 + 128, k0 - K0), B=(M, k0 + 128, k0), C=(M, k0 + 128, k0 + 128))


POTRF_INNER = [  # NBO, panel, rem, padding of lda
    (256, 0, 1, 0), (256, 0, 129, 2), (256, 0, 333, 2), (512, 0, 300, 0), (512, 0, 589, 2), (512, 2, 589, 0),
    (1024, 0, 1101, 0), (1024, 1, 1, 0), (1024, 3, 1101, 2), (1024, 6, 129, 0),
]


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('data', ['int', 'scaled'])
@pytest.mark.parametrize('nbo,panel,rem,pad', POTRF_INNER, ids=lambda v: str(v))
def test_caller_potrf_inner_update(lib, nbo, panel, rem, pad, data, kernel):
    """mode 1, tri 0, k = 128 < lda(A) = NBO, at column offsets 0 ... NBO - 256 of the workspace."""
    s = _potrf_inner(nbo, panel, rem, pad)
    assert s['n'] in (rem, nbo - 128 * (panel + 1)) and s['A'][2] <= nbo - 256
    _run(lib, kernel, data, s)


def _potrf_lazy(nbo, tiles, ragged, pad):
    """potrf_device, lazy update after the second outer block (K0 = NBO, K1 = 2 NBO): C += (-X) X^T on the lower
    triangle with A = all NBO columns of the workspace from row K1, B = columns K0 ... K1 and C = the trailing square
    of the matrix from row K1.  m = n = rem spans `tiles` row tiles, the last one partial (and rem odd) if ragged."""
    rem = 128 * tiles - (91 if ragged else 0)
    K0, K1 = nbo, 2 * nbo
    n_mat = K1 + rem
    W, M = Buf(n_mat + 1, nbo), Buf(n_mat + 1, _even(n_mat) + pad)
    return dict(m=rem, n=rem, k=nbo, mode=1, tri=1, A=(W, K1, 0), B=(M, K1, K0), C=(M, K1, K1))


# row tiles on both sides of the edges of the 8 x 8 super-tiles of the triangular raster
POTRF_LAZY = [(256, 1, True, 0), (512, 7, False, 2), (1024, 8, True, 0), (256, 9, False, 0), (512, 16, False, 0),
              (1024, 17, True, 2), (256, 24, True, 0), (512, 25, False, 2)]


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('data', ['int', 'scaled'])
@pytest.mark.parametrize('nbo,tiles,ragged,pad', POTRF_LAZY, ids=lambda v: str(v))
def test_caller_potrf_lazy_update(lib, nbo, tiles, ragged, pad, data, kernel):
    """mode 1, tri 1, k = NBO = lda(A)."""
    s = _potrf_lazy(nbo, tiles, ragged, pad)
    assert (s['m'] + T - 1) // T == tiles
    _run(lib, kernel, data, s)


def _trsm(m_l, k0, n_rows, pad):
    """trsm_right_lt_device after the column block at k0: X[:, k0 + 128:] += (-X_blk) L[k0 + 128:, k0 : k0 + 128]^T
    with A = the tight (n_rows x 128) workspace, B = a window of L (ldl > m) and C = a column window of X."""
    rest = m_l - k0 - 128
    Wn, L, X = Buf(n_rows + 1, 128), Buf(m_l + 1, m_l + 1 if m_l % 2 else m_l + 2), Buf(n_rows + 1, _even(m_l) + pad)
    return dict(m=n_rows, n=rest, k=128, mode=1, tri=0, A=(Wn, 0, 0), B=(L, k0 + 128, k0), C=(X, 0, k0 + 128))


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('data', ['int', 'scaled'])
@pytest.mark.parametrize('m_l,k0,n_rows,pad', [(351, 0, 65, 0), (351, 128, 4097, 2), (1107, 0, 1, 2), (1107, 896, 513, 0)],
                         ids=lambda v: str(v))
def test_caller_trsm_right_lt_update(lib, m_l, k0, n_rows, pad, data, kernel):
    """mode 1, tri 0, k = 128 = lda(A); n = the columns right of the block, odd here."""
    _run(lib, kernel, data, _trsm(m_l, k0, n_rows, pad))


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('data', ['int', 'scaled'])
@pytest.mark.parametrize('n_rows,m', [(33, 129), (1081, 129), (1081, 1100), (610, 2100)], ids=lambda v: str(v))
def test_caller_gram_tn(lib, n_rows, m, data, kernel):
    """sgdml_b200_gram_tn: C = Xt Xt^T, mode 0, beta 0, tri 1, with A and B the same pointer (the transposed factor,
    k = n_rows rounded up to even, not a multiple of 32) and a C that holds NaN and must not be read."""
    k = _even(n_rows)
    assert k % 32
    Xt, C = Buf(m + 1, k), Buf(m + 1, m + 1 if m % 2 else m + 2)
    _run(lib, kernel, data, dict(m=m, n=m, k=k, mode=0, alpha=1.0, beta=0.0, tri=1, A=(Xt, 0, 0), B=(Xt, 0, 0), C=(C, 0, 0)))


@pytest.mark.parametrize('kernel', TILE_KERNELS)
@pytest.mark.parametrize('data', ['int', 'scaled'])
@pytest.mark.parametrize('n_atoms,m_pad,n_rows', [(42, 200, 24), (42, 1000, 300), (100, 200, 36), (100, 1000, 129)], ids=lambda v: str(v))
def test_caller_predictor_large_d(lib, n_atoms, m_pad, n_rows, data, kernel):
    """run_queries for D > 256, with the padding of model_create: D = N (N - 1) / 2, DP = D rounded up to 8,
    DS = DP + 4 (868 = 4 mod 16 for 42 atoms, 4956 = 12 mod 16 for 100), Mpad = training points rounded up to 8; all
    strides tight.  S1 = Q Xc^T: mode 0, beta 0, k = DS, n = Mpad.  G = C1 XcT^T, then G += C2 JAT^T: mode 0, beta 0,
    then mode 1 into the same C with the beta = 0 the caller leaves in the arguments; k = Mpad, n = DP."""
    D = n_atoms * (n_atoms - 1) // 2
    DP = (D + 7) // 8 * 8
    DS = DP + 4
    assert DS % 16 == (4 if n_atoms == 42 else 12)
    Q, Xc, S1 = Buf(n_rows + 1, DS), Buf(m_pad + 1, DS), Buf(n_rows + 1, m_pad)
    _run(lib, kernel, data, dict(m=n_rows, n=m_pad, k=DS, mode=0, alpha=1.0, beta=0.0, A=(Q, 0, 0), B=(Xc, 0, 0), C=(S1, 0, 0)))
    C1, XcT, G = Buf(n_rows + 1, m_pad), Buf(DP + 1, m_pad), Buf(n_rows + 1, DP)
    first = dict(m=n_rows, n=DP, k=m_pad, mode=0, alpha=1.0, beta=0.0, A=(C1, 0, 0), B=(XcT, 0, 0), C=(G, 0, 0))
    g1 = _run(lib, kernel, data, first)
    C2, JAT = Buf(n_rows + 1, m_pad), Buf(DP + 1, m_pad)
    _run(lib, kernel, data, dict(first, mode=1, A=(C2, 0, 0), B=(JAT, 0, 0), seed=1), C0=g1)


# ================================================================================================ (d) the triangular raster
@pytest.mark.parametrize('kernel', TILE_KERNELS)
def test_triangular_raster_covers_every_tile_once(lib, kernel):
    """mode 1, tri 1 on C = 0 with A = B = ones (k = 2) at n = 20 000: 157 row tiles in 20 super-tile rows.  Every
    entry with col <= row is 2 (1 would be a tile the grid did not reach, 4 one it reached twice) and every tile above
    the diagonal keeps its NaN.  Checks the sqrt enumeration in the kernel against the block count of the launch;
    evaluated on the device, tile row by tile row."""
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < 8 << 30:
        pytest.skip('needs 8 GB of free device memory, %.1f GB are free' % (free / 2**30))
    n = 20000
    ones = Buf(n + 1, 2)
    ones.mat[:n] = 1.0
    C = torch.full((n, n), NAN, dtype=torch.float64, device='cuda')
    for ti in range((n + T - 1) // T):
        C[ti * T : (ti + 1) * T, : (ti + 1) * T] = 0.0
    canary = _bits(torch.full((1,), NAN, dtype=torch.float64, device='cuda'))[0]
    snap = ones.snapshot()
    _call(lib, kernel, n, n, 2, ones.ptr(), 2, ones.ptr(), 2, C.data_ptr(), n, mode=1, tri=1)
    _assert_unchanged(ones, snap, 'operands')
    wrong, written = [], []
    for ti in range((n + T - 1) // T):
        rows = C[ti * T : (ti + 1) * T]
        left, diag, right = rows[:, : ti * T], rows[:, ti * T : (ti + 1) * T], rows[:, (ti + 1) * T :]
        bad = torch.cat([left != 2.0, diag.tril() != torch.full_like(diag, 2.0).tril()], dim=1)
        if bool(bad.any()):
            wrong += [(ti, int(tj)) for tj in torch.unique(bad.nonzero()[:, 1] // T).tolist()]
        if right.numel() and bool((_bits(right) != canary).any()):
            written += [(ti, ti + 1 + int(tj)) for tj in torch.unique((_bits(right) != canary).nonzero()[:, 1] // T).tolist()]
    assert not wrong, 'tiles whose lower-triangle entries are not 2: %s' % wrong[:12]
    assert not written, 'tiles above the diagonal that were written: %s' % written[:12]


# ================================================================================================ (e) the abort flag
@pytest.mark.parametrize('kernel', ALL_KERNELS)
@pytest.mark.parametrize('tri', [0, 1], ids=['tri0', 'tri1'])
@pytest.mark.parametrize('form', ['mode0_general', 'mode1'])
def test_abort_flag(lib, form, tri, kernel):
    """A non-zero flag leaves all of C bit-identical; a zero flag gives the bits of the call without a flag."""
    import torch

    s = _plain_case(257, 257, 34, form, tri=tri)
    flags = torch.tensor([1, 0], dtype=torch.int32, device='cuda')
    hA, hB, hC0, _ = _case_data(257, 257, 34, 'scaled', False)
    A, B, C = s['A'][0], s['B'][0], s['C'][0]
    A.mat[:257, :34], B.mat[:257, :34], C.mat[:257, :257] = _up(hA), _up(hB), _up(hC0)
    snap = C.snapshot()
    args = (257, 257, 34, A.ptr(), A.ld, B.ptr(), B.ld, C.ptr(), C.ld, s['alpha'], s['beta'], s['mode'], tri)
    _call(lib, kernel, *args, flag=flags[0:].data_ptr())
    _assert_unchanged(C, snap, 'abort flag set')
    _call(lib, kernel, *args, flag=flags[1:].data_ptr())
    with_flag = C.snapshot()
    assert bool(C.changed(snap).any())  # the zero flag did not stop the call
    C.mat.copy_(snap)
    _call(lib, kernel, *args)
    _assert_unchanged(C, with_flag, 'zero flag against no flag')
    assert flags.tolist() == [1, 0]


# ================================================================================================ (f) determinism
@pytest.mark.parametrize('case', ['1025x257x1026_mode0_general', '300x300x130_mode1', '1100x1100x514_mode1_tri'])
def test_tile_kernels_are_deterministic_and_bit_identical(lib, case):
    """The same call twice gives the same bits, and the cp.async and TMA kernels give the same bits as each other:
    they share the tile shape, the fragment layout and the order of the k loop."""
    shape, form = case.split('_', 1)
    tri = int(form.endswith('_tri'))
    m, n, k = (int(x) for x in shape.split('x'))
    s = _plain_case(m, n, k, form.replace('_tri', ''), tri=tri)
    hA, hB, hC0, _ = _case_data(m, n, k, 'scaled', False)
    A, B, C = s['A'][0], s['B'][0], s['C'][0]
    A.mat[:m, :k], B.mat[:n, :k] = _up(hA), _up(hB)
    results = []
    for kernel in ('tma', 'tma', 'cpasync', 'cpasync'):
        C.mat[:m, :n] = _up(hC0)
        _call(lib, kernel, m, n, k, A.ptr(), A.ld, B.ptr(), B.ld, C.ptr(), C.ld, s['alpha'], s['beta'], s['mode'], tri)
        results.append(C.snapshot())
    for name, i, j in (('tma twice', 0, 1), ('cpasync twice', 2, 3), ('tma against cpasync', 0, 2)):
        diff = _bits(results[i]) != _bits(results[j])
        assert not bool(diff.any()), '%s: %d entries differ, first at %s' % (name, int(diff.sum()), diff.nonzero()[0].tolist())


# ================================================================================================ (g) offsets past 2^31 elements
WIDE_LD = 1 << 23  # 290 rows of this stride put the last row 2.4e9 elements from the first
WIDE_ROWS = 290


@pytest.fixture(scope='module')
def wide():
    """One 19.5 GB allocation, used as a 291-row matrix of row stride 2^23 whose leading columns alone are touched."""
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip('needs 24 GB of free device memory, %.1f GB are free' % (free / 2**30))
    storage = torch.empty((WIDE_ROWS + 1) * WIDE_LD, dtype=torch.float64, device='cuda')
    assert (WIDE_ROWS - 1) * WIDE_LD > 2**31
    yield storage
    del storage
    torch.cuda.empty_cache()


@pytest.mark.parametrize('kernel', ALL_KERNELS)
@pytest.mark.parametrize('form', ['mode0_beta1', 'mode1'])
@pytest.mark.parametrize('which', ['C', 'A', 'B'])
def test_wide_stride_gemm(lib, wide, which, form, kernel):
    """Exact integers with C, then A, then B in the matrix of row stride 2^23: every row * ld product of the kernels
    passes 2^31.  The wide operand has 290 rows, the other dimension 256; k = 64."""
    m, n, k = (256, WIDE_ROWS, 64) if which == 'B' else (WIDE_ROWS, 256, 64)
    s = _plain_case(m, n, k, form)
    cols = {'A': k, 'B': k, 'C': n}[which]
    s[which] = (Buf(WIDE_ROWS + 1, WIDE_LD, cols=cols + 16, storage=wide), 0, 0)
    _run(lib, kernel, 'int', s)


def _spd(n):
    G = np.random.default_rng(n).standard_normal((n, n))
    return G @ G.T / n + np.eye(n)


def test_wide_stride_potrf_potrs(lib, wide):
    """sgdml_b200_potrf and sgdml_b200_potrs (one and two right-hand sides) on a 290 x 290 matrix stored with
    lda = 2^23: k_potf2_tile, k_trsm_strip, both trailing updates and the k_trsv_* kernels index past 2^31."""
    import scipy.linalg

    n = WIDE_ROWS
    A = _spd(n)
    M = Buf(n + 1, WIDE_LD, cols=n + 16, storage=wide)
    M.mat[:n, :n] = _up(lc.nan_upper(np.tril(A)))
    snap = M.snapshot()
    _check(lib.sgdml_b200_potrf(M.ptr(), n, WIDE_LD, _stream()), 'potrf')
    _assert_unchanged(M, snap, 'potrf', (0, 0, n, n))
    lc.check_cholesky(A, M.mat[:n, :n].cpu().numpy(), forward_tol=1e-12)
    L = scipy.linalg.cholesky(A, lower=True)
    M.mat[:n, :n] = _up(lc.nan_upper(L))
    snap = M.snapshot()
    for nrhs in (1, 2):
        B0 = np.random.default_rng(nrhs).standard_normal((n, nrhs))
        Bd = _up(lc.with_padding(B0, nrhs + 3))
        _check(lib.sgdml_b200_potrs(M.ptr(), n, WIDE_LD, Bd.data_ptr(), nrhs, nrhs + 3, _stream()), 'potrs')
        X = Bd.cpu().numpy()
        lc.check_padding_unchanged(lc.with_padding(B0, nrhs + 3), X, nrhs, 'B')
        lc.check_potrs(A, L, B0, X, cond_ok=True)
    _assert_unchanged(M, snap, 'potrs (L is an input)')


def test_wide_stride_trsm_right_lt(lib, wide):
    """sgdml_b200_trsm_right_lt on 290 rows of X with ldx = 2^23 (three column blocks, the last partial)."""
    import scipy.linalg
    import torch

    n_rows, m = WIDE_ROWS, 290
    L = scipy.linalg.cholesky(_spd(m), lower=True)
    X0 = np.random.default_rng(5).standard_normal((n_rows, m))
    X = Buf(n_rows + 1, WIDE_LD, cols=m + 16, storage=wide)
    X.mat[:n_rows, :m] = _up(X0)
    Ld = _up(lc.nan_upper(L, m + 2))
    snap = X.snapshot()
    _check(lib.sgdml_b200_trsm_right_lt(Ld.data_ptr(), m, m + 2, X.ptr(), n_rows, WIDE_LD, _stream()), 'trsm_right_lt')
    torch.cuda.synchronize()
    _assert_unchanged(X, snap, 'trsm_right_lt', (0, 0, n_rows, m))
    lc.check_trsm_right_lt(L, X0, X.mat[:n_rows, :m].cpu().numpy(), cond_ok=True)
