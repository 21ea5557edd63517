"""The int8-slice GEMM k_ozaki_gemm<S> (csrc/ozaki.cu) in every slice count, raster and call shape its callers issue,
through the test hook sgdml_b200_ozaki_gemm_args, compared bit for bit with the exact model tests/ozaki_model.py.

Canaries.  A, B and C are windows of NaN-filled device buffers with padding columns and one more row after the last;
potrf's operands are windows of one n x lda matrix.  Everything outside the write set (the whole window of C, or with
tri = 1 the 128 x 32 tiles (tm, tn) with 32 tn <= 128 tm + 127) must keep its bits, and with overwrite = 1 the window of
C keeps its NaN: it must not be read.

A result is compared with `==` on the bits (NaN against NaN, whatever its payload, counts as equal).  A failure names
the 128 x 32 tiles that differ and, for the first differing entry, the level or slice pair whose loss or duplication
explains the difference when one does.  Large shapes compute the model's integer level sums with a device FP64 matmul,
which is exact for them (every partial sum is an integer below 2^31)."""

import numpy as np
import pytest

import ozaki_model as om
from test_gemm_classes import Buf, _bits

pytestmark = pytest.mark.gpu

NAN = float('nan')
BM, BN = om.BM, om.BN


@pytest.fixture(autouse=True)
def _no_debug_flags(monkeypatch):
    """SGDML_B200_OZAKI_DBG switches parts of the kernel off."""
    monkeypatch.delenv('SGDML_B200_OZAKI_DBG', raising=False)


@pytest.fixture(scope='module')
def lib():
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return _lib.lib()


def _stream():
    from sgdml_b200 import _lib

    return _lib.current_stream()


def _up(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _call(lib, m, n, k, alpha, A, lda, B, ldb, C, ldc, S, tri=0, overwrite=0):
    import torch

    from sgdml_b200 import _lib

    rc = lib.sgdml_b200_ozaki_gemm_args(m, n, k, alpha, A, lda, B, ldb, C, ldc, S, tri, overwrite, _stream())
    _lib.check(rc, 'ozaki_gemm_args')
    torch.cuda.synchronize()


def _device_levels(sa, sb, S):
    """om.levels with the products on the device (exact: integer operands, partial sums below 2^31)."""
    import torch

    ta = _up(sa)
    tb = ta if sb is sa else _up(sb)
    out = []
    for L in range(2, S + 2):
        acc = None
        for p, q in om.level_pairs(S, L):
            t = ta[p - 1] @ tb[q - 1].T
            acc = t if acc is None else acc + t
        out.append(acc.cpu().numpy())
    return out


def _model(hA, hB, C_old, alpha, S, overwrite, tri, same):
    m, n, k = hA.shape[0], hB.shape[0], hA.shape[1]
    big = m * n * k * S > 1 << 27
    lev = om.operands(hA, hA if same else hB, S, _device_levels if big else None)
    return om.gemm(hA, hB, C_old, alpha, S, overwrite=bool(overwrite), tri=bool(tri), lev=lev)


def _assert_unchanged(buf, snap, what, window=None, may_write=None):
    """Every entry of buf keeps its bits, except, inside window = (r0, c0, m, n), those may_write (a bool m x n device
    mask; None = the whole window) allows."""
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
        rel = (' = (%d, %d) of the window of C, 128 x 32 tile (%d, %d)' % (r - r0, c - c0, (r - r0) // BM, (c - c0) // BN)
               if window else '')
        raise AssertionError('%s: %d entries outside the write set were written; first at (%d, %d) of the buffer%s'
                             % (what, int(changed.sum()), r, c, rel))


def _compare(got, want, mask, what, hA=None, hB=None, alpha=1.0, S=7, C_old=None):
    same = (got.view(np.int64) == want.view(np.int64)) | (np.isnan(got) & np.isnan(want))
    bad = ~same & mask
    if bad.any():
        i, j = (int(x) for x in np.argwhere(bad)[0])
        why = ''
        if hA is not None and C_old is not None:
            base = 0.0 if np.isnan(C_old[i, j]) else C_old[i, j]
            why = '; ' + om.explain(hA, hB, alpha, S, got[i, j] - base, want[i, j] - base, i, j)
        raise AssertionError('%s: %d entries differ from the exact model, in 128 x 32 tiles %s; first at (%d, %d): %r, '
                             'expected %r%s' % (what, int(bad.sum()), om.tiles_of(bad), i, j, float(got[i, j]),
                                                float(want[i, j]), why))


def _run(lib, s, hA, hB, hC0=None):
    """One call as the dict s describes it: m, n, k, S, alpha, overwrite, tri and A, B, C = (Buf, first row, first column).
    Fills the windows (C0 goes into the write set unless the call overwrites), calls, checks that nothing outside the
    write set changed and that the result equals the model bit for bit, and returns the result."""
    import torch

    m, n, k, S = s['m'], s['n'], s['k'], s['S']
    alpha, overwrite, tri = s.get('alpha', 1.0), s.get('overwrite', 0), s.get('tri', 0)
    same = s['A'] == s['B']
    (Ab, ar, ac), (Bb, br, bc), (Cb, cr, cc) = s['A'], s['B'], s['C']
    Ab.mat[ar : ar + m, ac : ac + k] = _up(hA)
    if not same:
        Bb.mat[br : br + n, bc : bc + k] = _up(hB)
    mask = om.tri_mask(m, n) if tri else np.ones((m, n), dtype=bool)
    if not overwrite:
        c = hC0 if not tri else np.where(mask, hC0, NAN)
        Cb.mat[cr : cr + m, cc : cc + n] = _up(c)
    C_old = Cb.mat[cr : cr + m, cc : cc + n].cpu().numpy()
    bufs = {id(b): b for b in (Ab, Bb, Cb)}
    snaps = {i: b.snapshot() for i, b in bufs.items()}
    _call(lib, m, n, k, alpha, Ab.ptr(ar, ac), Ab.ld, Bb.ptr(br, bc), Bb.ld, Cb.ptr(cr, cc), Cb.ld, S, tri, overwrite)
    what = 'S %d %dx%dx%d alpha %g overwrite %d tri %d' % (S, m, n, k, alpha, overwrite, tri)
    for i, b in bufs.items():
        if b is Cb:
            dmask = torch.from_numpy(mask).cuda() if tri else None
            _assert_unchanged(b, snaps[i], what, (cr, cc, m, n), dmask)
        else:
            _assert_unchanged(b, snaps[i], what + ' (operand buffer)')
    del snaps
    got = Cb.mat[cr : cr + m, cc : cc + n].cpu().numpy()
    want = _model(hA, hA if same else hB, C_old, alpha, S, overwrite, tri, same)
    _compare(got, want, mask, what, hA, hA if same else hB, alpha, S, C_old)
    return got


def _plain(m, n, k, S, alpha=1.0, overwrite=0, tri=0, same=False):
    """Separate buffers with padding columns and a NaN row after the last (A == B when same)."""
    A = Buf(m + 1, k + 3)
    B = A if same else Buf(n + 1, k + 5)
    C = Buf(m + 1, n + 2)
    return dict(m=m, n=n, k=k, S=S, alpha=alpha, overwrite=overwrite, tri=tri, A=(A, 0, 0), B=(B, 0, 0), C=(C, 0, 0))


def _normal(m, n, k, seed=0, row_exp=3):
    """Standard-normal operands with rows scaled by 2^e, |e| <= row_exp, and a C0 of the product's size."""
    rng = np.random.default_rng([m, n, k, seed])
    ea = rng.integers(-row_exp, row_exp + 1, size=(m, 1))
    eb = rng.integers(-row_exp, row_exp + 1, size=(n, 1))
    A = np.ldexp(rng.standard_normal((m, k)), ea)
    B = np.ldexp(rng.standard_normal((n, k)), eb)
    C0 = np.ldexp(rng.standard_normal((m, n)) * np.sqrt(k), ea + eb.T)
    return A, B, C0


def test_hook_rejects_what_it_cannot_launch(lib):
    """Slice counts outside 2..7, k outside 1..16384, strides shorter than a row, host or null pointers, tri on a
    non-square C and tri or overwrite outside {0, 1} are argument errors, reported before anything is launched: C keeps
    its bits."""
    import torch

    A, B, C = Buf(9, 8), Buf(9, 8), Buf(9, 8)
    A.mat[:], B.mat[:], C.mat[:] = 1.0, 1.0, 3.0
    snap = C.snapshot()
    host = np.ones((9, 8))
    ok = dict(m=8, n=8, k=8, A=A.ptr(), lda=8, B=B.ptr(), ldb=8, C=C.ptr(), ldc=8, S=7, tri=0, overwrite=0)
    bad = [dict(S=1), dict(S=8), dict(S=0), dict(k=0), dict(k=16385, lda=16385, ldb=16385), dict(lda=6), dict(ldb=6),
           dict(ldc=6), dict(A=host.ctypes.data), dict(B=host.ctypes.data), dict(C=host.ctypes.data), dict(A=None),
           dict(tri=1, m=6), dict(tri=2), dict(overwrite=2), dict(overwrite=-1), dict(m=0), dict(n=0)]
    for change in bad:
        a = dict(ok, **change)
        rc = lib.sgdml_b200_ozaki_gemm_args(a['m'], a['n'], a['k'], 1.0, a['A'], a['lda'], a['B'], a['ldb'], a['C'],
                                            a['ldc'], a['S'], a['tri'], a['overwrite'], _stream())
        assert rc == -1000, change  # SGDML_B200_ERR_ARG
    torch.cuda.synchronize()
    _assert_unchanged(C, snap, 'rejected calls')


# ================================================================================================ the edge grid
M_EDGES = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257]  # the two 64-row warpgroup halves and the 128-row tiles
N_EDGES = [1, 31, 32, 33, 63, 64, 65, 127, 128, 129]  # 32-column tiles
K_EDGES = [1, 63, 64, 65, 127, 128, 129, 255, 256, 257]  # 64-wide k-blocks, k padded to 128
GRID = sorted(
    {(M_EDGES[i], N_EDGES[(3 * i + 5) % 10], K_EDGES[(7 * i + 1) % 10]) for i in range(10)}
    | {(M_EDGES[(3 * i + 1) % 10], N_EDGES[i], K_EDGES[i]) for i in range(10)}
    | {(257, 129, 257), (1, 1, 1)}
)
GRID_REDUCED = GRID[::3]
FORMS = {'acc': (1.0, 0), 'neg_over': (-1.0, 1), 'a0.3_acc': (0.3, 0), 'a0.3_over': (0.3, 1)}


def _shape_id(c):
    return '%dx%dx%d' % c


def test_grid_covers_every_edge():
    assert {c[0] for c in GRID} == set(M_EDGES) and {c[1] for c in GRID} == set(N_EDGES)
    assert {c[2] for c in GRID} == set(K_EDGES)


@pytest.mark.parametrize('form', sorted(FORMS))
@pytest.mark.parametrize('shape', GRID, ids=_shape_id)
def test_edge_grid_seven_slices(lib, shape, form):
    alpha, overwrite = FORMS[form]
    _run(lib, _plain(*shape, 7, alpha, overwrite), *_normal(*shape))


@pytest.mark.parametrize('form', ['acc', 'neg_over'])
@pytest.mark.parametrize('shape', GRID_REDUCED, ids=_shape_id)
@pytest.mark.parametrize('S', [2, 3, 4, 5, 6])
def test_edge_grid_every_slice_count(lib, S, shape, form):
    alpha, overwrite = FORMS[form]
    _run(lib, _plain(*shape, S, alpha, overwrite), *_normal(*shape, seed=S))


# the shapes of the former tolerance tests: FP64 comparisons at S = 7, rows scaled by 2^+-20 with alpha = -1, a
# symmetric tri update, and S = 4..7 on one shape
BRINGUP = {
    'fp64_128x64x128': dict(m=128, n=64, k=128, S=7),
    'fp64_128x64x256': dict(m=128, n=64, k=256, S=7),
    'fp64_256x128x128': dict(m=256, n=128, k=128, S=7),
    'fp64_300x200x130': dict(m=300, n=200, k=130, S=7),
    'fp64_129x65x1000': dict(m=129, n=65, k=1000, S=7),
    'fp64_64x8x40': dict(m=64, n=8, k=40, S=7),
    'row_scaling_200x136x384': dict(m=200, n=136, k=384, S=7, alpha=-1.0, row_exp=20),
    'tri_384x384x256': dict(m=384, n=384, k=256, S=7, alpha=-1.0, tri=1),
    'slices4_256x192x512': dict(m=256, n=192, k=512, S=4),
    'slices5_256x192x512': dict(m=256, n=192, k=512, S=5),
    'slices6_256x192x512': dict(m=256, n=192, k=512, S=6),
    'slices7_256x192x512': dict(m=256, n=192, k=512, S=7),
}


@pytest.mark.parametrize('overwrite', [0, 1])
@pytest.mark.parametrize('case', sorted(BRINGUP))
def test_exact_bringup_shapes(lib, case, overwrite):
    c = BRINGUP[case]
    m, n, k, S, tri = c['m'], c['n'], c['k'], c['S'], c.get('tri', 0)
    A, B, C0 = _normal(m, n, k, row_exp=c.get('row_exp', 3))
    _run(lib, _plain(m, n, k, S, c.get('alpha', 1.0), overwrite, tri, same=bool(tri)), A, A if tri else B, C0)


# ================================================================================================ persistence
PERSIST = [(1000, S) for S in range(2, 8)] + [(64, 2), (64, 7), (128, 4), (128, 6)]


@pytest.mark.parametrize('k,S', PERSIST, ids=lambda v: str(v))
def test_persistent_walk(lib, k, S):
    """2200 x 2200: 69 x 69 tiles of 128 x 32 in 3 x 3 super-tiles of 1024 x 1024, many tiles per CTA, so the stage
    ring (3 to 8 stages by S) wraps across tile boundaries with its phases carried over."""
    m = n = 2200
    _run(lib, _plain(m, n, k, S, -1.0), *_normal(m, n, k, seed=S))


# ================================================================================================ tri
@pytest.mark.parametrize('n,same,overwrite', [(1, True, 0), (33, True, 0), (127, True, 0), (128, True, 0),
                                              (129, True, 0), (1025, True, 0), (2049, True, 0), (129, False, 0),
                                              (1025, True, 1), (2049, False, 0)], ids=lambda v: str(v))
def test_tri(lib, n, same, overwrite):
    """Whole 128 x 32 tiles reaching the lower triangle are written (above the diagonal too); no other entry is."""
    A, B, C0 = _normal(n, n, 200, seed=n)
    _run(lib, _plain(n, n, 200, 7, -1.0, overwrite, tri=1, same=same), A, A if same else B, C0)


def test_triangular_raster_writes_every_kept_tile_once(lib):
    """tri at n = 20 000 (157 tile rows, 20 super-tile rows) with all-ones rows, k = 2, alpha = -1 and C = 0 on the
    write set: every kept entry is exactly -2 (0 would be a tile the raster missed, -4 one it visited twice) and every
    other entry keeps its NaN.  Evaluated on the device, tile row by tile row."""
    import torch

    free, _ = torch.cuda.mem_get_info()
    if free < 8 << 30:
        pytest.skip('needs 8 GB of free device memory, %.1f GB are free' % (free / 2**30))
    n, k = 20000, 2
    ones = Buf(n + 1, k)
    ones.mat[:n] = 1.0
    C = torch.full((n, n), NAN, dtype=torch.float64, device='cuda')
    for tm in range((n + BM - 1) // BM):  # the write set: 32 tn <= 128 tm + 127, i.e. columns below 128 (tm + 1)
        C[tm * BM : (tm + 1) * BM, : (tm + 1) * BM] = 0.0
    canary = _bits(torch.full((1,), NAN, dtype=torch.float64, device='cuda'))[0]
    snap = ones.snapshot()
    _call(lib, n, n, k, -1.0, ones.ptr(), k, ones.ptr(), k, C.data_ptr(), n, 7, tri=1)
    _assert_unchanged(ones, snap, 'operands')
    wrong, written = [], []
    for tm in range((n + BM - 1) // BM):
        rows = C[tm * BM : (tm + 1) * BM]
        kept, right = rows[:, : (tm + 1) * BM], rows[:, (tm + 1) * BM :]
        bad = kept != -float(k)
        if bool(bad.any()):
            wrong += [(tm, int(tn)) for tn in torch.unique(bad.nonzero()[:, 1] // BN).tolist()]
        if right.numel() and bool((_bits(right) != canary).any()):
            cols = (_bits(right) != canary).nonzero()[:, 1]
            written += [(tm, (tm + 1) * BM // BN + int(tn)) for tn in torch.unique(cols // BN).tolist()]
    assert not wrong, '128 x 32 tiles whose kept entries are not -%d: %s' % (k, wrong[:12])
    assert not written, '128 x 32 tiles outside the write set that were written: %s' % written[:12]


# ================================================================================================ the callers' call shapes
# potrf's lazy update after the second outer block (K0 = NBO, K1 = 2 NBO): C -= X X^T with X = A[K1:, K0:K1] and
# C = A[K1:, K1:], both windows of the one (n x lda) matrix, split once; rem = n - K1 rows.  (rem, NBO, lda - n, S)
POTRF = [(1, 256, 0, 7), (127, 512, 1, 6), (128, 1024, 0, 7), (129, 256, 1, 6), (1000, 512, 0, 7),
         (3000, 1024, 1, 7), (3000, 256, 0, 6), (1000, 1024, 1, 6), (129, 1024, 0, 7)]


@pytest.mark.parametrize('rem,nbo,pad,S', POTRF, ids=lambda v: str(v))
def test_caller_potrf_lazy_update(lib, rem, nbo, pad, S):
    K0, K1 = nbo, 2 * nbo
    n_mat = K1 + rem
    M = Buf(n_mat + 1, n_mat + pad)
    rng = np.random.default_rng([rem, nbo, pad, S])
    X = rng.standard_normal((rem, nbo)) / np.sqrt(nbo)
    C0 = rng.standard_normal((rem, rem))
    s = dict(m=rem, n=rem, k=nbo, S=S, alpha=-1.0, overwrite=0, tri=1, A=(M, K1, K0), B=(M, K1, K0), C=(M, K1, K1))
    _run(lib, s, X, X, C0)


# run_queries for D > 256 with model_create's padding: D = N (N - 1) / 2, DP = D rounded up to 8, DS = DP + 4 (so
# DS = 4 mod 8), Mpad = training points rounded up to 8, every stride tight.  (N, Mpad, rows of the batch, slices)
PREDICT = [(24, 40, 127, 4), (30, 104, 128, 5), (60, 200, 129, 6), (100, 48, 255, 5), (181, 40, 257, 4),
           (181, 64, 129, 6)]


@pytest.mark.parametrize('n_atoms,m_pad,n_rows,S', PREDICT, ids=lambda v: str(v))
def test_caller_predictor_contractions(lib, n_atoms, m_pad, n_rows, S):
    """S1 = Q Xc^T and S2 = Q JA^T (k = DS, n = Mpad, overwrite), then G = C1 XcT^T (overwrite) and G += C2 JAT^T into the
    same G (k = Mpad, n = DP).  N = 181 gives DS = 16 300, near the limit of 16 384."""
    D = n_atoms * (n_atoms - 1) // 2
    DP = (D + 7) // 8 * 8
    DS = DP + 4
    assert DS % 8 == 4 and DS <= om.K_MAX
    rng = np.random.default_rng([n_atoms, m_pad, n_rows, S])
    Q = rng.uniform(0.05, 1.0, size=(n_rows, DS))  # descriptors (inverse distances), padding columns included
    Xc = rng.standard_normal((m_pad, DS)) * 0.1
    JA = np.ldexp(rng.standard_normal((m_pad, DS)), rng.integers(-12, 0, size=(m_pad, 1)))
    Qb, Xb, Jb = Buf(n_rows + 1, DS), Buf(m_pad + 1, DS), Buf(m_pad + 1, DS)
    for name, Bb, hB in (('S1', Xb, Xc), ('S2', Jb, JA)):
        Sb = Buf(n_rows + 1, m_pad)
        _run(lib, dict(m=n_rows, n=m_pad, k=DS, S=S, overwrite=1, A=(Qb, 0, 0), B=(Bb, 0, 0), C=(Sb, 0, 0)), Q, hB)
    C1 = rng.standard_normal((n_rows, m_pad))
    C2 = np.ldexp(rng.standard_normal((n_rows, m_pad)), rng.integers(-8, 8, size=(n_rows, 1)))
    XcT, JAT = np.ascontiguousarray(Xc[:, :DP].T), np.ascontiguousarray(JA[:, :DP].T)
    G = Buf(n_rows + 1, DP)
    first = dict(m=n_rows, n=DP, k=m_pad, S=S, overwrite=1, A=(Buf(n_rows + 1, m_pad), 0, 0),
                 B=(Buf(DP + 1, m_pad), 0, 0), C=(G, 0, 0))
    g1 = _run(lib, first, C1, XcT)
    _run(lib, dict(first, overwrite=0, A=(Buf(n_rows + 1, m_pad), 0, 0), B=(Buf(DP + 1, m_pad), 0, 0)), C2, JAT, g1)


# ================================================================================================ limits and operand rows
def test_longest_contraction_is_exact(lib):
    """k = 16 384 (256 k-blocks), with rows of entries just below their maximum, whose first slices are all +-64 and
    whose level sums are the largest the data allow; k = 16 385 is rejected (test_hook_rejects_what_it_cannot_launch)."""
    m, n, k = 130, 70, om.K_MAX
    A, B, C0 = _normal(m, n, k)
    rng = np.random.default_rng(5)
    A[::4] = np.where(rng.random((len(A[::4]), k)) < 0.5, -1.0, 1.0) * (1 - 2.0**-53)
    B[::3] = np.where(rng.random((len(B[::3]), k)) < 0.5, -1.0, 1.0) * (1 - 2.0**-53)
    _run(lib, _plain(m, n, k, 7, -1.0), A, B, C0)


def _special_rows(case, m, n, k, seed):
    A, B, C0 = _normal(m, n, k, seed=seed, row_exp=0)
    rng = np.random.default_rng(seed)
    if case == 'zero_and_single':
        A[0] = A[5] = A[129] = 0.0
        A[5, 17] = 3.5
        B[0] = B[33] = B[64] = 0.0
        B[33, k - 1] = -2.0**-5
    elif case == 'rows_2^20':
        A = np.ldexp(A, np.where(np.arange(m) % 2, 20, -20)[:, None])
        B = np.ldexp(B, np.where(np.arange(n) % 3, -20, 20)[:, None])
    elif case == 'rows_2^1000':  # products of 2^2000 overflow, of 2^-2000 vanish, others land in the subnormal range
        A = np.ldexp(A, np.array([1000, -1000, 0])[np.arange(m) % 3][:, None])
        B = np.ldexp(B, np.array([-1000, 1000, 0, -20])[np.arange(n) % 4][:, None])
    elif case == 'max_2^1023':  # e = 1025: 2^e alone is not a double
        A[0, 3] = 2.0**1023
        A[1] = np.ldexp(A[1], 1000)
        A[1, 0] = -(2.0**1023)
        A[2] = 2.0**1023 * (1 - 2.0**-53) * np.where(rng.random(k) < 0.5, -1, 1)
        B[0] = 0.0
        B[1:40] = np.ldexp(B[1:40], -1060)
        B[40:50] = np.ldexp(B[40:50], -30)
    elif case == 'max_2^-1030':  # 2^-e alone is not a double; the rows are subnormal
        A[0] = np.ldexp(A[0], -1060)
        A[0, 0] = 2.0**-1030
        A[1] = 0.0
        A[1, 7] = 2.0**-1030
        A[2] = np.ldexp(np.rint(A[2] * 64), -1074)  # multiples of the smallest subnormal
        B[:10] = np.ldexp(B[:10], 1000)
    elif case == 'ties':  # entries on the half-way grid 2^-(7p + 1) of the slicing: rint's ties to even
        p = rng.integers(1, 8, size=(m, k))
        A = rng.integers(-60, 61, size=(m, k)) / 128.0 + np.where(rng.random((m, k)) < 0.5, -1, 1) * 2.0 ** (-7 * p - 1)
        A[:, 0] = 0.45
        B[1::2] = rng.integers(-64, 65, size=B[1::2].shape) / 256.0 + 2.0**-9
    elif case == 'nan_inf_in_a':
        A[3, 7], A[130, 0], A[64, k - 1] = NAN, np.inf, -np.inf
    elif case == 'nan_inf_in_b':
        B[0, 5], B[31, 100], B[32, 0] = NAN, np.inf, -np.inf
    else:
        raise ValueError(case)
    return A, B, C0


ROW_CASES = ['zero_and_single', 'rows_2^20', 'rows_2^1000', 'max_2^1023', 'max_2^-1030', 'ties', 'nan_inf_in_a',
             'nan_inf_in_b']


@pytest.mark.parametrize('S', [3, 7])
@pytest.mark.parametrize('case', ROW_CASES)
def test_operand_rows(lib, case, S):
    """Zero and single-entry rows, rows scaled by 2^+-20 and 2^+-1000, row maxima of 2^1023 and 2^-1030, rounding ties,
    and NaN / +-Inf, which make their row (in A) or column (in B) of C NaN."""
    m, n, k = 150, 70, 140
    A, B, C0 = _special_rows(case, m, n, k, S)
    got = _run(lib, _plain(m, n, k, S, -1.0), A, B, C0)
    if case.startswith('nan_inf'):
        assert np.isnan(got).any() and not np.isnan(got).all()


# ================================================================================================ determinism
def test_repeated_calls_are_bit_identical(lib):
    m, n, k, S = 1100, 700, 600, 6
    A, B, C0 = _normal(m, n, k)
    s = _plain(m, n, k, S, 0.3)
    first = _run(lib, s, A, B, C0)
    (Ab, _, _), (Bb, _, _), (Cb, _, _) = s['A'], s['B'], s['C']
    for _ in range(2):
        Cb.mat[:m, :n] = _up(C0)
        _call(lib, m, n, k, 0.3, Ab.ptr(), Ab.ld, Bb.ptr(), Bb.ld, Cb.ptr(), Cb.ld, S)
        again = Cb.mat[:m, :n].cpu().numpy()
        assert np.array_equal(again.view(np.int64), first.view(np.int64))


@pytest.mark.parametrize('n', [129, 700])
def test_tri_matches_full_product_on_its_tiles(lib, n):
    """With A == B the tri call and the full call give the same bits on every tile the tri call writes."""
    k, S = 300, 7
    A, _, C0 = _normal(n, n, k)
    full = _run(lib, _plain(n, n, k, S, -1.0, same=True), A, A, C0)
    tri = _run(lib, _plain(n, n, k, S, -1.0, tri=1, same=True), A, A, C0)
    mask = om.tri_mask(n, n)
    assert np.array_equal(full[mask].view(np.int64), tri[mask].view(np.int64))


# ================================================================================================ the slice setting
def test_solve_slices_below_two_mean_fp64(lib, monkeypatch):
    """SGDML_B200_OZAKI_SLICES=1 (and 0, and negative values) select the FP64 trailing updates: potrf gives the FP64
    factor bit for bit and get_solve_slices reports 0."""
    import torch

    from sgdml_b200 import _lib

    assert lib.sgdml_b200_set_solve_slices(-1) == 0
    n = 3000
    rng = np.random.default_rng(1)
    G = rng.standard_normal((n, n // 4))
    A = G @ G.T + 1e-3 * np.eye(n)
    outs = {}
    for mode in ('0', '1', '-3'):
        monkeypatch.setenv('SGDML_B200_OZAKI_SLICES', mode)
        assert lib.sgdml_b200_get_solve_slices() == 0
        Ad = _up(A)
        _lib.check(lib.sgdml_b200_potrf(Ad.data_ptr(), n, n, _stream()), 'potrf')
        torch.cuda.synchronize()
        outs[mode] = np.tril(Ad.cpu().numpy())
    assert np.array_equal(outs['1'], outs['0']) and np.array_equal(outs['-3'], outs['0'])
