"""Kernel-matrix assembly in every routing class against the oracle, entry by entry (tests/assemble_checks.py).

Each class of assemble_checks.CLASSES first confirms through the engine's plan query that it runs in its class, then
checks the full square matrix (with its mirrored blocks), a seeded column subset, a row range, several row launches
and a row range from m_begin = 1 in launches of one row point against the componentwise bound; one class per kernel
adds a host K with padding columns and scale = -1.  The energy-constraint kernels run at atom counts around the warp
edges of their per-warp reduction.  Every output buffer starts as NaN, so an entry no launch writes cannot pass on a
previous call's values.  The oracle is computed once per shape and sliced."""

import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import assemble_checks as ac  # noqa: E402
from oracle import assemble as oassemble  # noqa: E402
from oracle import desc as odesc  # noqa: E402

PER_KERNEL = ('v4_tj8', 'v5_full', 'large_gmem', 'k_tj')  # the classes that also run the host-K and scale = -1 cases


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


@pytest.fixture(scope='module')
def n_sm(eng):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope='module')
def problem():
    """Problem of a class shape with its oracle K and magnitudes, computed once per shape."""
    from sgdml_b200 import synth

    cache = {}

    def get(case):
        key = (case.N, case.rot, case.swap, case.M, case.sig)
        if key not in cache:
            perms = synth.rotor_swap_group(case.N, case.rot, case.swap)
            R = synth.geometries(case.N, case.M, 2).reshape(case.M, -1)
            x, g = (np.ascontiguousarray(a) for a in odesc.from_R(R))  # the C ABI takes C-contiguous arrays
            lin = odesc.tril_perms_lin(perms)
            cache[key] = dict(x=x, g=g, lin=lin, K=oassemble.assemble(x, g, lin, case.sig),
                              scale=ac.assemble_abs_scale(x, g, lin, case.sig))
        return cache[key]

    return get


@contextlib.contextmanager
def _hooks(*variants):
    from sgdml_b200 import _lib

    L = _lib.lib()
    try:
        for v in variants:
            assert L.sgdml_b200_set_assemble_variant(v) == 0
        yield
    finally:
        L.sgdml_b200_set_assemble_variant(1000 + 65535)
        L.sgdml_b200_set_assemble_variant(0)


def _subset(N, M, seed):
    """Every column point, each without one whole atom and without a random third of the other columns."""
    rng = np.random.default_rng(seed)
    n3 = 3 * N
    keep = rng.random((M, n3)) > 0.3
    drop = rng.integers(0, N, size=M)
    keep[np.arange(M)[:, None], 3 * drop[:, None] + np.arange(3)[None, :]] = False
    keep[np.arange(M), 3 * ((drop + 1) % N)] = True  # at least one column per point
    return np.nonzero(keep.ravel())[0].astype(np.int64)


def _assemble(t, args, N, M, cols=None, rows=None, scale=1.0):
    """sgdml_b200_assemble_rows into a device buffer filled with NaN: an entry no launch writes fails every check (a
    fresh torch.empty buffer may reuse a block that still holds the previous call's correct values)."""
    import torch

    lo, hi = (0, M) if rows is None else rows
    n_cols = 3 * N * M if cols is None else len(cols)
    K = torch.full(((hi - lo) * 3 * N, (n_cols + 1) // 2 * 2), float('nan'), dtype=torch.float64, device='cuda')
    t._assemble_kernel_mat_device(*args, col_idxs=cols, rows=rows, scale=scale, out=K)
    return K[:, :n_cols].cpu().numpy()


def _launch_cap(M):
    """Row points per launch that do not divide M."""
    return next(r for r in range(2, M + 1) if M % r)


def _same_launch(p, q):
    return (p.kernel, p.TJ, p.PG, p.n_chunks) == (q.kernel, q.TJ, q.PG, q.n_chunks)


def _upper_blocks(K, n3):
    iu = np.triu_indices(K.shape[0])
    blk = (iu[0] // n3) <= (iu[1] // n3)
    return K[iu][blk]


@pytest.mark.parametrize('name', list(ac.CLASSES))
def test_class_vs_oracle(eng, problem, n_sm, name):
    from sgdml_b200 import _lib

    case = ac.CLASSES[name]
    pr = problem(case)
    N, M, S, sig = case.N, case.M, ac.n_perms(case), case.sig
    n3, n = 3 * N, 3 * N * case.M
    x, g, lin, K_ref, scale = pr['x'], pr['g'], pr['lin'], pr['K'], pr['scale']
    k = ac.n_terms(N, S)
    t = eng.GDMLTrain()
    args = (x, g, lin, sig)
    worst = {}

    def check(K, rows, cols, what, m_begin=0):
        ref = K_ref[rows][:, cols]
        worst[what] = ac.check_K(K, ref, scale[rows][:, cols], k, what='%s %s' % (name, what), n_atoms=N,
                                 cols=np.arange(n)[cols], m_begin=m_begin)

    def in_class(nk, nJ, nr, square):
        p = ac.plan(N, S, nk, nJ, nr, square, n_sm)
        assert case.cls in ac.classes_of(p, N, S, nJ, nr, n_sm), (name, p)
        return p

    allr, allc = np.s_[:], np.s_[:]
    with _hooks(case.variant):
        # full square matrix: sym mirrors the upper block triangle, bit for bit
        p_full = in_class(N, M, M, True)
        K = _assemble(t, args, N, M)
        check(K, allr, allc, 'full')
        if p_full.sym:
            for i in range(M):
                for j in range(i + 1, M):
                    assert np.array_equal(K[j * n3:(j + 1) * n3, i * n3:(i + 1) * n3],
                                          K[i * n3:(i + 1) * n3, j * n3:(j + 1) * n3].T), (name, i, j)
        # seeded column subset: NK < N, a partial last tile of column points
        cols = _subset(N, M, seed=N + M)
        nJ, nk = ac.col_shape(cols, N)
        assert nk < N and nJ == M
        p_cols = in_class(nk, nJ, M, False)
        assert p_cols.TJ == 1 or nJ % p_cols.TJ
        nc = len(cols)
        Kc = _assemble(t, args, N, M, cols=cols)
        check(Kc, allr, cols, 'cols')
        # row range: all columns, and the column subset bit for bit against the same rows of the call above
        lo, hi = 1, M - 1
        in_class(N, M, hi - lo, False)
        Kr = _assemble(t, args, N, M, rows=(lo, hi))
        check(Kr, np.s_[lo * n3:hi * n3], allc, 'rows', m_begin=lo)
        assert _same_launch(in_class(nk, nJ, hi - lo, False), p_cols)
        Krc = _assemble(t, args, N, M, cols=cols, rows=(lo, hi))
        assert np.array_equal(Krc, Kc[lo * n3:hi * n3])
    r = _launch_cap(M)
    with _hooks(case.variant, 1000 + r):
        # several row launches of r row points (r does not divide M): no mirroring, the same blocks as one launch
        p_multi = in_class(N, M, M, True)
        large = p_multi.kernel == 'k_assemble_large'  # one launch takes every row point
        assert p_multi.sym == 0 and p_multi.rows_per_launch == (M if large else r)
        Km = _assemble(t, args, N, M)
        check(Km, allr, allc, 'launches of %d rows' % r)
        assert _same_launch(p_multi, p_full)
        assert np.array_equal(_upper_blocks(Km, n3), _upper_blocks(K, n3))
    with _hooks(case.variant, 1001):
        # a row range from m_begin = 1 in launches of one row point each: every launch starts at its own row point
        p_one = in_class(N, M, M - 1, False)
        assert p_one.sym == 0 and p_one.rows_per_launch == (M - 1 if large else 1)
        Kro = _assemble(t, args, N, M, rows=(1, M))
        check(Kro, np.s_[n3:], allc, 'rows 1.. in launches of 1 row', m_begin=1)
        assert _same_launch(p_one, p_multi)
        assert np.array_equal(Kro, Km[n3:])
    if name in PER_KERNEL:
        with _hooks(case.variant):
            # host K with padding columns (ldk > n_cols) for a column subset
            ldk = nc + 3
            Kh = np.full((n, ldk), np.nan)
            L = _lib.lib()
            _lib.check(L.sgdml_b200_assemble_rows(
                _lib.ptr(x), _lib.ptr(g), _lib.ptr(lin), N, M, S, float(sig), _lib.ptr(cols), nc, 1.0, 0, M,
                Kh.ctypes.data, ldk, _lib.current_stream()), 'assemble')
            check(np.ascontiguousarray(Kh[:, :nc]), allr, cols, 'host K, ldk %d' % ldk)
            # scale = -1, the sign the analytic solver factorises
            Kn = _assemble(t, args, N, M, scale=-1.0)
            assert np.array_equal(Kn, -K)
            check(-Kn, allr, allc, 'scale -1')
    if name == 'k_tj':
        # k_assemble_large keeps k_assemble's summation order: bit-identical where both compute a block directly
        with _hooks(1):
            p_large = ac.plan(N, S, nk, nJ, M, False, n_sm)
            assert p_large.kernel == 'k_assemble_large' and p_large.grid_x < M * nJ  # CTAs walk several blocks
            Kl = _assemble(t, args, N, M, cols=cols)
            Klf = _assemble(t, args, N, M)
        assert p_cols.kernel == 'k_assemble'
        assert np.array_equal(Kl, Kc)
        assert np.array_equal(_upper_blocks(Klf, n3), _upper_blocks(K, n3))
    print('\n[assemble bound] %-12s %-58s max |err| / (tau scale): %s  (tau %.2e)'
          % (name, case.cls, ', '.join('%s %.2e' % kv for kv in worst.items()), ac.tau(k)))


@pytest.mark.parametrize('N', [31, 32, 33, 64, 65, 129])
def test_ecstr_warp_edges_vs_oracle(eng, N):
    """k_assemble_ecstr and k_assemble_ecstr_rows run one thread per atom in whole warps and reduce |delta|^2 through
    one slot per warp: 1, 1, 2, 2, 3 and 5 warps here, the last one partial except at 32 and 64."""
    import torch

    from sgdml_b200 import _lib, synth

    M = 3 if N < 100 else 2
    sig = 40
    perms = synth.rotor_swap_group(N, 1, 0)
    S = len(perms)
    x, g = (np.ascontiguousarray(a) for a in odesc.from_R(synth.geometries(N, M, 5).reshape(M, -1)))
    lin = odesc.tril_perms_lin(perms)
    K_ref = oassemble.assemble_E_cstr(x, g, lin, sig)
    scale = ac.ecstr_full_scale(x, g, lin, sig)
    k = ac.n_terms(N, S)
    n3, n = 3 * N, 3 * N * M
    t = eng.GDMLTrain()
    L = _lib.lib()
    args = (_lib.ptr(x), _lib.ptr(g), _lib.ptr(lin), N, M, S, float(sig))
    # every output buffer starts as NaN: an entry no kernel writes fails the check
    ldk = (n + M + 1) // 2 * 2
    K = torch.full((n + M, ldk), float('nan'), dtype=torch.float64, device='cuda')
    t._assemble_kernel_mat_device(x, g, lin, sig, out=K[:n])
    _lib.check(L.sgdml_b200_assemble_ecstr(*args, 1.0, K.data_ptr(), ldk, _lib.current_stream()), 'assemble_ecstr')
    w_full = ac.check_K(K[:, :n + M].cpu().numpy(), K_ref, scale, k, what='ecstr N %d' % N)
    # rows: the force rows of points [lo, M), then their energy rows; columns: some force columns and every energy one
    rng = np.random.default_rng(N)
    cols = np.concatenate([np.unique(rng.integers(0, n, size=2 * N)), n + np.arange(M)])
    nc, lo = len(cols), 1
    rows = np.concatenate([np.arange(lo * n3, n), n + np.arange(lo, M)])
    Kr = torch.full(((M - lo) * (n3 + 1), nc + 1), float('nan'), dtype=torch.float64, device='cuda')
    _lib.check(L.sgdml_b200_assemble_ecstr_rows(*args, _lib.ptr(cols), nc, 1.0, lo, M, Kr.data_ptr(), nc + 1,
                                                _lib.current_stream()), 'assemble_ecstr_rows')
    w_rows = ac.check_K(Kr[:, :nc].cpu().numpy(), K_ref[rows][:, cols], scale[rows][:, cols], k,
                        what='ecstr_rows N %d' % N)
    print('\n[assemble bound] ecstr N %d (%d warps): max |err| / (tau scale) full %.2e, rows %.2e  (tau %.2e)'
          % (N, -(-N // 32), w_full, w_rows, ac.tau(k)))
