"""The acceptance checks of tests/assemble_checks.py on CPU: the engine's assembly plan (a host-only query) against the
conditions the kernels rely on over a grid of shapes and every hook state, the class table against the plan, and the
componentwise bound on K against the oracle -- it passes an independent FP64 evaluation and fails each injected
defect, including defects the older normwise check (rel_err < 1e-12) accepts.  No GPU needed."""

import ctypes as C
import itertools

import numpy as np
import pytest

import assemble_checks as ac
from conftest import rel_err
from oracle import assemble as oassemble
from oracle import desc as odesc

_ERR_ARG = -1000  # SGDML_B200_ERR_ARG (include/sgdml_b200.h)


@pytest.fixture
def lib():
    from sgdml_b200 import _lib

    L = _lib.lib()
    yield L
    L.sgdml_b200_set_assemble_variant(0)
    L.sgdml_b200_set_assemble_variant(1000 + 65535)


# ------------------------------------------------------------------------------------------------ plan query
def test_plan_query_arguments(lib):
    out = (C.c_int64 * 10)()
    f = lib.sgdml_b200_assemble_plan
    assert f(9, 6, 9, 45, 45, 1, 132, out) == 0
    assert ac.plan(9, 6, 9, 45, 45, True) == ac.Plan('k_assemble_v4', 8, 6, 1, 2, 79836, 1, 65535, 0, 0)
    for bad in [
        (1, 6, 1, 4, 4, 1, 132),  # one atom
        (1024, 6, 1024, 4, 4, 1, 132),  # N^2 beyond the fast-division range
        (9, 0, 9, 4, 4, 1, 132),  # no permutation
        (9, 6, 0, 4, 4, 0, 132),  # no kept column atom
        (9, 6, 10, 4, 4, 0, 132),  # more kept column atoms than atoms
        (9, 6, 9, 0, 4, 0, 132),  # no column point
        (9, 6, 9, 4, 0, 0, 132),  # no row point
        (9, 6, 8, 4, 4, 1, 132),  # square with a column subset
        (9, 6, 9, 4, 3, 1, 132),  # square over part of the rows
        (9, 6, 9, 4, 4, 2, 132),
        (9, 6, 9, 4, 4, 1, 0),  # no SM
        (9, 6, 9, 2 ** 31, 4, 0, 132),
    ]:
        assert f(*bad, out) == _ERR_ARG, bad
    assert f(9, 6, 9, 4, 4, 1, 132, None) == _ERR_ARG


def test_plan_follows_the_hooks(lib):
    assert ac.plan(9, 6, 9, 10, 10, True).kernel == 'k_assemble_v4'
    lib.sgdml_b200_set_assemble_variant(2)
    assert ac.plan(9, 6, 9, 10, 10, True).kernel == 'k_assemble'
    lib.sgdml_b200_set_assemble_variant(5)
    assert ac.plan(9, 6, 9, 10, 10, True).kernel == 'k_assemble_v5'
    lib.sgdml_b200_set_assemble_variant(1)
    assert ac.plan(9, 6, 9, 10, 10, True).kernel == 'k_assemble_large'
    lib.sgdml_b200_set_assemble_variant(0)
    lib.sgdml_b200_set_assemble_variant(1003)
    p = ac.plan(9, 6, 9, 10, 10, True)
    assert p.rows_per_launch == 3 and p.sym == 0  # several launches: no mirrored stores
    assert ac.plan(9, 6, 9, 10, 3, False).rows_per_launch == 3


_HOOKS = [(kernel, large, rows) for kernel in (0, 2, 4, 5) for large in (0, 1) for rows in (65535, 3)]
_SIZES = [(45, 45, True), (7, 3, False), (200, 70000, False)]  # (column points, row points, square)
_S = (1, 2, 3, 6, 12, 20, 81, 120, 243)


def _set_hooks(lib, kernel, large, rows):
    lib.sgdml_b200_set_assemble_variant(0)
    if kernel:
        assert lib.sgdml_b200_set_assemble_variant(kernel) == 0
    if large:
        assert lib.sgdml_b200_set_assemble_variant(1) == 0
    assert lib.sgdml_b200_set_assemble_variant(1000 + rows) == 0


@pytest.mark.parametrize('kernel,large,rows', _HOOKS)
def test_plan_invariants(lib, kernel, large, rows):
    """Over N = 2...1023, nine permutation counts, three kept-column counts and three grid sizes: what each kernel
    needs of its launch.  Read off the kernels in csrc/assemble.cu:
      * dynamic shared memory within the 227 KB of an sm_90 CTA;
      * grid.y (row points per launch of the grid.y kernels) and grid.z at most 65535;
      * every (column point, row atom, kept column atom) sub-block of a tile has a thread: the item index
        blockIdx.z * 1024 + tid + q * 256 covers TJ N NK, with TJ N^2 <= 1024 whenever TJ > 1 (no grid.z then);
      * grid.x covers every column point without empty CTAs (v4 / v5: groups of 4 tiles; k_assemble: one tile);
      * v4 / v5 only for N <= 255 (byte permutation tables), 1 <= PG <= S, TJ PG <= 256 (one thread per
        (column point, permutation) slot forms the Matern factors);
      * sym only for the full square matrix in one launch (the mirrored store addresses absolute row points), never
        for k_assemble_large;
      * k_assemble_large: the delta table in shared memory only within 100 KB (two CTAs per SM), and the slabs of all
        CTAs within 2 GB unless a single CTA runs."""
    _set_hooks(lib, kernel, large, rows)
    f = lib.sgdml_b200_assemble_plan
    out = (C.c_int64 * 10)()
    par, res = [], []
    for N, S in itertools.product(range(2, 1024), _S):
        for nk in sorted({1, -(-N // 3), N}):
            for nJ, nr, sq in _SIZES:
                if sq and nk != N:
                    continue
                assert f(N, S, nk, nJ, nr, int(sq), 132, out) == 0
                par.append((N, S, nk, nJ, nr, sq))
                res.append(tuple(out))
    N, S, NK, nJ, nr, sq = np.array(par, dtype=np.int64).T
    kern, TJ, PG, z, gx, smem, sym, rpl, slab, dl = np.array(res, dtype=np.int64).T
    small = kern < 3
    tiled = (kern == 1) | (kern == 2)

    def need(cond, what):
        bad = np.nonzero(~cond)[0]
        assert bad.size == 0, '%s fails at %d shapes, first (N, S, NK, nJ, rows, square) = %s: plan %s' % (
            what, bad.size, par[bad[0]], res[bad[0]])

    need(smem <= 227 * 1024, 'shared memory <= 227 KB')
    need(~small | ((rpl >= 1) & (rpl <= 65535) & (rpl == rows)), 'grid.y <= 65535')
    need((z >= 1) & (z <= 65535), 'grid.z <= 65535')
    need(~small | (z * 1024 >= TJ * N * NK), 'a thread for every sub-block')
    need(~small | (TJ == 1) | ((TJ * N * N <= 1024) & (z == 1)), 'TJ N^2 <= 1024 when TJ > 1')
    need(~small | ((TJ >= 1) & (TJ <= np.minimum(8, nJ))), '1 <= TJ <= min(8, nJ)')
    tiles = -(-nJ // TJ)
    need(~tiled | ((gx * 4 >= tiles) & ((gx - 1) * 4 < tiles)), 'v4 / v5 grid.x: ceil(tiles / 4)')
    need((kern != 0) | (gx == tiles), 'k_assemble grid.x: one tile per CTA')
    need(~tiled | (N <= 255), 'v4 / v5 only for N <= 255')
    need(~tiled | ((PG >= 1) & (PG <= S) & (TJ * PG <= 256)), '1 <= PG <= S, TJ PG <= 256')
    need((kern != 2) | (TJ == 1), 'v5 runs one column point per tile')
    need((sym == 0) | ((sq == 1) & (rpl >= nr)), 'sym only for the square matrix in one launch')
    need((kern != 3) | (sym == 0), 'k_assemble_large never mirrors')
    need((kern != 3) | ((gx >= 1) & (gx <= np.minimum(nr * nJ, 2 * 132))), 'k_assemble_large grid.x')
    need((kern != 3) | (dl == 0) | (8 * N * N <= 100 * 1024), 'delta table in shared memory within 100 KB')
    need((kern != 3) | (smem == np.where(dl == 1, 8 * N * N, 0)), 'k_assemble_large shared memory = its delta table')
    need((kern != 3) | (gx == 1) | (slab * 8 * gx <= 2 << 30), 'slabs within 2 GB')
    need((kern == 3) | ((slab == 0) & (dl == 0)), 'slab and delta table only for k_assemble_large')
    if large:
        need(kern == 3, 'variant 1 runs k_assemble_large')
    elif kernel == 2:
        need(kern != 1, 'variant 2 never runs v4')


# ------------------------------------------------------------------------------------------------ classes
def _class_plan(lib, case, n_sm=ac.H100_SMS):
    lib.sgdml_b200_set_assemble_variant(case.variant)
    try:
        return ac.plan(case.N, ac.n_perms(case), case.N, case.M, case.M, True, n_sm)
    finally:
        lib.sgdml_b200_set_assemble_variant(0)


def test_every_class_is_tested(lib):
    """Each named shape lands in its class, and together they reach every class the routing has: deleting the only
    shape of a class, or a routing change that moves a shape out of its class, fails here."""
    reached = set()
    for name, case in list(ac.CLASSES.items()) + [('slab_capped', ac.SLAB_CAPPED)]:
        p = _class_plan(lib, case)
        got = ac.classes_of(p, case.N, ac.n_perms(case), case.M, case.M)
        assert case.cls in got, (name, case, p, got)
        reached |= {case.cls}
    assert reached == ac.DOCUMENTED
    p = _class_plan(lib, ac.SLAB_CAPPED)  # 214 CTAs of 10 MB at N = 370, S = 3 on 132 SMs
    assert (p.kernel, p.grid_x, p.dl_in_smem) == ('k_assemble_large', 214, 0) and p.slab * 8 * p.grid_x <= 2 << 30


# ------------------------------------------------------------------------------------------------ the bound
@pytest.fixture(scope='module')
def fx():
    """Seven atoms, S = 6, four training points, the last one compressed to 0.6 of its size and sig = 0.1: the blocks
    between it and the others are ~1e-15 of max |K|, so a defect confined to them passes rel_err < 1e-12."""
    from sgdml_b200 import synth

    N, M, sig = 7, 4, 0.1
    perms = synth.rotor_swap_group(N, 1, 1)
    R = synth.geometries(N, M, 3)
    R[-1] *= 0.6
    x, g = odesc.from_R(R.reshape(M, -1))
    lin = odesc.tril_perms_lin(perms)
    K = oassemble.assemble(x, g, lin, sig)
    return dict(N=N, M=M, S=len(perms), sig=sig, x=x, g=g, lin=lin, perms=perms, K=K,
                scale=ac.assemble_abs_scale(x, g, lin, sig), k=ac.n_terms(N, len(perms)))


def _blk(f, i, j):
    n3 = 3 * f['N']
    return np.s_[i * n3:(i + 1) * n3, j * n3:(j + 1) * n3]


def _rejected(f, K):
    """The older normwise check accepts K, check_K does not."""
    assert rel_err(K, f['K']) < 1e-12
    with pytest.raises(AssertionError, match='outside tau'):
        ac.check_K(K, f['K'], f['scale'], f['k'], n_atoms=f['N'])


def test_t_abs_is_the_dense_product(fx):
    t = ac._Terms(fx['x'], fx['g'], fx['lin'], fx['sig'])
    assert np.array_equal(t.P, fx['perms'])
    J = np.abs(odesc.d_desc_from_comp(fx['g']))
    dense = np.stack([J[0].T @ J[3][tp] for tp in t.tp])
    assert rel_err(t.t_abs(0, 3), dense) < 1e-15


def test_scale_dominates_the_result(fx):
    assert np.all(np.abs(fx['K']) <= fx['scale'])
    assert np.max(fx['scale'][_blk(fx, 0, 3)]) < 1e-13 * np.max(np.abs(fx['K']))  # the fixture's tiny blocks


def test_subsets_of_the_scale(fx):
    n3 = 3 * fx['N']
    cols = np.array([0, 5, n3 + 1, 3 * n3 - 1, 3 * n3, 4 * n3 - 2])
    s = ac.assemble_abs_scale(fx['x'], fx['g'], fx['lin'], fx['sig'], cols=cols, rows=(1, 3))
    ref = fx['scale'][n3:3 * n3][:, cols]
    assert np.all(np.abs(s - ref) <= 1e-14 * ref)  # the same sums, BLAS may block them differently


def test_independent_fp64_evaluation_passes(fx):
    """The oracle's closed form (SURVEY.md section 8 row a-K: a different summation order) agrees within the bound."""
    x, g, N, M = fx['x'], fx['g'], fx['N'], fx['M']
    tp = odesc.tril_perms_from_lin(fx['lin'], fx['S'])
    K2 = np.block([[oassemble.kernel_block(x[i], g[i], x[j], g[j], tp, fx['sig']) for j in range(M)] for i in range(M)])
    ratio = ac.check_K(K2, fx['K'], fx['scale'], fx['k'], n_atoms=N)
    assert 0 < ratio < 1


def test_one_entry_perturbed_fails(fx):
    K = fx['K'].copy()
    b = _blk(fx, 0, 3)
    r, c = np.unravel_index(np.argmax(fx['scale'][b]), fx['scale'][b].shape)
    K[b][r, c] += 10 * ac.tau(fx['k']) * fx['scale'][b][r, c]
    _rejected(fx, K)


def test_small_entry_with_the_wrong_sign_fails(fx):
    K = fx['K'].copy()
    small = np.abs(K) < 1e-13 * np.max(np.abs(K))  # < 1e-6 max |K|, and a sign flip keeps rel_err < 1e-12
    ratio = np.where(small, np.abs(K) / fx['scale'], 0.0)
    r, c = np.unravel_index(np.argmax(ratio), K.shape)
    K[r, c] = -K[r, c]
    _rejected(fx, K)


def test_transposed_sub_block_fails(fx):
    K = fx['K'].copy()
    blk = K[_blk(fx, 0, 3)]
    N = fx['N']
    sub = blk.reshape(N, 3, N, 3).transpose(0, 2, 1, 3)  # [a, b] = 3 x 3 sub-block
    asym = np.abs(sub - sub.transpose(0, 1, 3, 2)).sum(axis=(2, 3))
    a, b = np.unravel_index(np.argmax(asym), asym.shape)
    blk[3 * a:3 * a + 3, 3 * b:3 * b + 3] = blk[3 * a:3 * a + 3, 3 * b:3 * b + 3].T.copy()
    _rejected(fx, K)


def test_dropped_permutation_fails(fx):
    K = fx['K'].copy()
    x, g = fx['x'], fx['g']
    tp = odesc.tril_perms_from_lin(fx['lin'], fx['S'])
    K[_blk(fx, 0, 3)] = oassemble.kernel_block(x[0], g[0], x[3], g[3], np.delete(tp, 2, axis=0), fx['sig'])
    _rejected(fx, K)


def test_mirrored_block_not_transposed_fails(fx):
    K = fx['K'].copy()
    K[_blk(fx, 3, 0)] = K[_blk(fx, 0, 3)]
    _rejected(fx, K)


def test_nan_fails(fx):
    K = fx['K'].copy()
    K[1, 2] = np.nan
    with pytest.raises(AssertionError, match=r'block \(0, 0\), entry \(1, 2\)'):
        ac.check_K(K, fx['K'], fx['scale'], fx['k'], n_atoms=fx['N'])


def test_energy_constraint_scale(fx):
    """The energy-constraint magnitudes dominate the oracle's entries, and a K_fe or K_ee entry of the tiny pair moved
    by 10 tau scale fails."""
    x, g, lin, sig = fx['x'], fx['g'], fx['lin'], fx['sig']
    K = oassemble.assemble_E_cstr(x, g, lin, sig)
    s = ac.ecstr_full_scale(x, g, lin, sig)
    assert np.all(np.abs(K) <= s)
    n, t = 3 * fx['N'] * fx['M'], ac.tau(fx['k'])
    for r, c in [(n + 0, 3 * 3 * fx['N'] + 4), (4, n + 3), (n + 3, n + 0)]:
        assert s[r, c] < 1e-13 * np.max(np.abs(K))
        K2 = K.copy()
        K2[r, c] += 10 * t * s[r, c]
        assert rel_err(K2, K) < 1e-12
        with pytest.raises(AssertionError):
            ac.check_K(K2, K, s, fx['k'])
