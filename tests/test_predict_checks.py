"""The acceptance checks of tests/predict_checks.py on CPU: the chunk plan against hand-computed plans, and the
componentwise force / energy bound against the oracle -- on a plain, an energy-constrained and a periodic model it
passes an independent FP64 evaluation and fails each injected defect of the kind a multi-chunk prediction could have,
plus defects specific to energy constraints and to cells.  The persistent main kernel's schedule (main_schedule) against
hand-computed schedules at 132 and 114 SMs, its tile classes against the kernel source, and the bound against the
outputs of four schedule faults in one query tile.  No GPU needed."""

import numpy as np
import pytest

import predict_checks as pc
from oracle import desc as odesc
from oracle import predict as opredict


# ------------------------------------------------------------------------------------------------ chunk plans
def _plan(n_atoms, n_train, S, B, host_io, **kw):
    ly = pc.layout(n_atoms, n_train)
    return pc.chunk_plan(ly.D, ly.DP, ly.Mpad, S, ly.large, B, host_io, **kw)


def test_layout():
    assert pc.layout(9, 200) == pc.Layout(36, 40, 64, 32, 224, False)
    assert pc.layout(21, 1000) == pc.Layout(210, 224, 32, 16, 1008, False)
    assert pc.layout(23, 19) == pc.Layout(253, 256, 32, 8, 24, False)
    assert pc.layout(24, 29) == pc.Layout(276, 280, 8, 8, 32, True)
    assert pc.layout(42, 2000) == pc.Layout(861, 864, 8, 8, 2000, True)
    assert pc.layout(60, 3000) == pc.Layout(1770, 1776, 8, 8, 3000, True)


def test_chunk_plan_aspirin():
    # 2^28 / (224 * 8) / 6 = 24 966 queries per chunk
    assert pc.chunk_geos(224, 1008, 6, False) == 24966
    dev = _plan(21, 1000, 6, 65536, False)
    assert dev.chunks == [(0, 24966), (24966, 49932), (49932, 65536)]
    assert dev.slots == [0, 0, 0] and not dev.pipelined and not dev.graph and dev.main_launches == 3
    host = _plan(21, 1000, 6, 65536, True)
    assert host.chunks == [(0, 16384), (16384, 32768), (32768, 49152), (49152, 65536)]
    assert host.slots == [0, 1, 0, 1] and host.pipelined and host.main_launches == 4
    assert pc.edge_rows(dev) == [0, 24965, 24966, 49931, 49932, 65535]


def test_chunk_plan_ethanol():
    assert pc.chunk_geos(40, 224, 6, False) == 65536  # the 65 536 cap applies
    assert _plan(9, 200, 6, 65536, False).chunks == [(0, 65536)]
    assert _plan(9, 200, 6, 65536, True).chunks == [(i * 16384, (i + 1) * 16384) for i in range(4)]
    tail = _plan(9, 200, 6, 3 * 65536 + 3, False)
    assert tail.chunks == [(0, 65536), (65536, 131072), (131072, 196608), (196608, 196611)]
    assert tail.main_launches == 4
    h4096 = _plan(9, 200, 6, 4096, True)
    assert h4096.chunks == [(0, 1024), (1024, 2048), (2048, 3072), (3072, 4096)] and h4096.slots == [0, 1, 0, 1]
    h4095 = _plan(9, 200, 6, 4095, True)  # one chunk on the caller's stream
    assert h4095.chunks == [(0, 4095)] and not h4095.pipelined and h4095.main_launches == 1
    h4097 = _plan(9, 200, 6, 4097, True)  # max(1024, ceil(4097 / 4)) = 1025
    assert h4097.chunks == [(0, 1025), (1025, 2050), (2050, 3075), (3075, 4097)]
    g16 = _plan(9, 200, 6, 16, True)
    assert g16.graph and g16.chunks == [(0, 16)] and g16.main_launches == 0
    g17 = _plan(9, 200, 6, 17, True)
    assert not g17.graph and g17.chunks == [(0, 17)] and g17.main_launches == 1
    assert not _plan(9, 200, 6, 16, False).graph  # device buffers never take the graph path
    assert _plan(9, 200, 6, 0, True).chunks == []


def test_chunk_plan_large_descriptors():
    # ac-ala3-nhme: min(2^31 / (864 * 8), 2^31 / (2000 * 8)) / 243 = 552
    assert pc.chunk_geos(864, 2000, 243, True) == 552
    p = _plan(42, 2000, 243, 4096, False)
    assert len(p.chunks) == 8 and p.chunks[-1] == (3864, 4096) and p.main_launches == 16
    # c60, I_h: 89 478 / 120 = 745; K.v over 3000 training points is 4 chunks of 745 and a tail of 20
    assert pc.chunk_geos(1776, 3000, 120, True) == 745
    t = _plan(60, 3000, 120, 3000, True, train=True)
    assert t.chunks == [(0, 745), (745, 1490), (1490, 2235), (2235, 2980), (2980, 3000)]
    assert not t.pipelined and not t.graph and t.main_launches == 10


def test_chunk_cap_hook_arguments():
    """sgdml_b200_set_predict_chunk is host code: it runs without a GPU.  Negative caps are rejected."""
    from sgdml_b200 import _lib

    L = _lib.lib()
    try:
        assert L.sgdml_b200_set_predict_chunk(-1) == -1000
        assert 'max_geos >= 0' in _lib.last_error()
        assert L.sgdml_b200_set_predict_chunk(7) == 0
    finally:
        assert L.sgdml_b200_set_predict_chunk(0) == 0


def test_chunk_plan_cap():
    p = _plan(9, 200, 6, 4097, True, cap=7)  # hundreds of alternating chunks
    assert len(p.chunks) == 586 and p.chunks[-1] == (4095, 4097)
    assert p.slots[:4] == [0, 1, 0, 1] and p.slots[-1] == 1 and p.main_launches == 586
    assert _plan(9, 200, 6, 23, False, cap=7).chunks == [(0, 7), (7, 14), (14, 21), (21, 23)]
    assert _plan(24, 29, 6, 23, False, cap=5).main_launches == 10
    assert _plan(21, 40, 6, 1, False, cap=1).chunks == [(0, 1)]
    assert _plan(9, 200, 6, 7, True, cap=2).graph  # the graph path runs the batch whole, whatever the cap


# ------------------------------------------------------------------------------------------------ the bound
N, M, SIG, B = 9, 50, 20, 40  # M = 50: the last 32-point training tile is partially padded (18 real points)
CAP = 16
KINDS = ('plain', 'ecstr', 'pbc')  # energy constraints in the kernel; a periodic model in the skewed cell
AE_SCALE = 0.05


def _model(M_=M, reverse=False, kind='plain'):
    from sgdml_b200 import synth

    perms = synth.rotor_swap_group(N, 1, 1)
    R = synth.geometries(N, M, 0).reshape(M, -1)
    alphas = np.random.default_rng(99).standard_normal((M, 3 * N))
    lat = pc.skewed_cell(N) if kind == 'pbc' else None
    x, g = odesc.from_R(R, None if lat is None else (lat, np.linalg.inv(lat)))
    ja = odesc.d_desc_dot_vec(g, alphas)
    ae = AE_SCALE * np.random.default_rng(98).standard_normal(M)
    x, ja, ae = x[:M_], ja[:M_], ae[:M_]
    if reverse:
        x, ja, ae = x[::-1], ja[::-1], ae[::-1]
    model = {
        'type': 'm',
        'z': np.ones(N, dtype=np.int64),
        'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': np.ascontiguousarray(ja),
        'c': 0.37,
        'std': 1.7,
        'sig': SIG,
        'perms': perms,
        'tril_perms_lin': odesc.tril_perms_lin(perms),
    }
    if kind == 'ecstr':
        model['alphas_E'] = np.ascontiguousarray(ae)
    if lat is not None:
        model['lattice'] = lat
    return model


_CASES = {}


def _case(kind):
    from sgdml_b200 import synth

    if kind not in _CASES:
        model = _model(kind=kind)
        op = opredict.Predictor(model)
        R = synth.geometries(N, B, 1).reshape(B, -1)
        if kind == 'pbc':
            assert np.min(pc.pbc_margin(R, *op.lat_and_inv)) >= 1e-6
        E, F = op.predict(R)
        scale = pc.predict_abs_scale(model, R, oracle=op)
        k = pc.n_terms(M, op.n_perms, N * (N - 1) // 2)
        plan = _plan(N, M, op.n_perms, B, False, cap=CAP)
        assert plan.chunks == [(0, 16), (16, 32), (32, 40)]
        _CASES[kind] = dict(kind=kind, model=model, op=op, R=R, E=E, F=F, scale=scale, k=k, plan=plan)
    return _CASES[kind]


@pytest.fixture(scope='module')
def cases():
    """The plain, energy-constrained and periodic cases: every generic check below runs on all three."""
    return [_case(kind) for kind in KINDS]


@pytest.fixture(scope='module')
def ecstr_case():
    return _case('ecstr')


@pytest.fixture(scope='module')
def pbc_case():
    return _case('pbc')


def test_tau_at_aspirin_shape():
    assert pc.tau(pc.n_terms(1000, 6, 210)) < 1e-11


def test_scale_dominates_the_result(cases):
    for case in cases:
        sE, sF = case['scale']
        assert np.all(sF >= np.abs(case['F']) * (1 - 1e-12)) and np.all(sE > 0)
        assert np.all(sE >= np.abs(case['E'] - 0.37) * (1 - 1e-12))


def _longdouble_desc(R, lat):
    """Periodic descriptors evaluated in np.longdouble and rounded once to FP64 (the same images: no query is near a
    tie)."""
    ld = np.longdouble
    r = np.asarray(R, dtype=ld).reshape(R.shape[0], -1, 3)
    a, b = np.tril_indices(r.shape[1], -1)
    d = r[:, a, :] - r[:, b, :]
    L, Li = np.asarray(lat, dtype=ld), np.asarray(np.linalg.inv(lat), dtype=ld)
    k = np.round(np.einsum('ij,...j->...i', Li, d))
    d = d - np.einsum('ij,...j->...i', L, k)
    dist = np.sqrt(np.sum(d * d, axis=-1))
    return (1 / dist).astype(np.float64), (d / (dist ** 3)[..., None]).astype(np.float64)


def _predict_desc(model, x, g):
    """The oracle's prediction from given query descriptors (its R=None path)."""
    op = opredict.Predictor(model)
    op.set_R_desc(x)
    op.set_R_d_desc(g)
    return op.predict()


def test_independent_fp64_evaluation_passes(cases):
    """The training points in reverse order: every sum runs in another order, so the rounding differs.  The periodic
    case takes its query descriptors from an np.longdouble evaluation."""
    for case in cases:
        rev = _model(reverse=True, kind=case['kind'])
        if case['kind'] == 'pbc':
            E2, F2 = _predict_desc(rev, *_longdouble_desc(case['R'], rev['lattice']))
        else:
            E2, F2 = opredict.Predictor(rev).predict(case['R'])
        assert not np.array_equal(F2, case['F'])
        rF, rE = pc.check_predict(E2, F2, case['E'], case['F'], case['scale'], case['k'])
        assert rF < pc.tau(case['k']) / 10 and rE < pc.tau(case['k']) / 10
        pc.check_predict(None, F2, None, case['F'], case['scale'], case['k'])  # return_E=False


def _fails(case, E, F, match=None):
    with pytest.raises(AssertionError, match=match):
        pc.check_predict(E, F, case['E'], case['F'], case['scale'], case['k'])


def test_chunk_shifted_by_one_geometry_fails(cases):
    for case in cases:
        lo, hi = case['plan'].chunks[1]
        E, F = case['E'].copy(), case['F'].copy()
        F[lo:hi] = case['F'][lo + 1 : hi + 1]
        E[lo:hi] = case['E'][lo + 1 : hi + 1]
        _fails(case, E, F, 'force entries')


def test_stale_chunk_fails(cases):
    """One chunk holds the previous call's outputs (another batch of the same size)."""
    from sgdml_b200 import synth

    for case in cases:
        E_prev, F_prev = case['op'].predict(synth.geometries(N, B, 2).reshape(B, -1))
        lo, hi = case['plan'].chunks[2]
        E, F = case['E'].copy(), case['F'].copy()
        F[lo:hi], E[lo:hi] = F_prev[lo:hi], E_prev[lo:hi]
        _fails(case, E, F)


def test_dropped_term_fails(cases):
    """One (training point, permutation) term missing from one geometry's sums."""
    for case in cases:
        op = case['op']
        S = op.n_perms
        k_drop = (M - 1) * S + S - 1  # last training point, last permutation
        sub = opredict.Predictor(case['model'])
        sub.R_desc_perms = np.delete(op.R_desc_perms, k_drop, axis=0)
        sub.R_d_desc_alpha_perms = np.delete(op.R_d_desc_alpha_perms, k_drop, axis=0)
        if op.alphas_E_lin is not None:
            sub.alphas_E_lin = np.delete(op.alphas_E_lin, k_drop)
        i = 21
        E_i, F_i = sub.predict(case['R'][i : i + 1])
        E, F = case['E'].copy(), case['F'].copy()
        E[i], F[i] = E_i[0], F_i[0]
        _fails(case, E, F, 'force entries')
        _fails(case, E, case['F'], 'energies')  # the energy alone gives it away too


def test_dropped_padded_tile_fails(cases):
    """The last, partially padded 32-point training tile (points 32..49) missing from every sum."""
    for case in cases:
        ly = pc.layout(N, M)
        assert ly.BM == 32 and ly.Mpad == 64 and M % ly.BM != 0
        E, F = opredict.Predictor(_model(M_=M - M % ly.BM, kind=case['kind'])).predict(case['R'])
        _fails(case, E, F, 'force entries')


def test_one_entry_perturbed_fails(cases):
    for case in cases:
        sF = case['scale'][1]
        F = case['F'].copy()
        F[29, 17] += 1e-10 * sF[29, 17]
        _fails(case, case['E'], F, r'first at \(29, 17\)')


def test_nan_fails(cases):
    for case in cases:
        F = case['F'].copy()
        F[39, 0] = np.nan
        _fails(case, case['E'], F)
        E = case['E'].copy()
        E[3] = np.nan
        _fails(case, E, case['F'])


# ------------------------------------------------------------------------------------------------ energy constraints
def _norms(op, R_desc):
    """n = sqrt5 |q - x_k| (B, M S) for query descriptors R_desc (B, D)."""
    diff = np.asarray(R_desc)[:, None, :] - op.R_desc_perms[None]
    return np.sqrt(5.0) * np.sqrt(np.sum(diff * diff, axis=-1))


def test_alphas_E_dropped_for_one_point_fails(ecstr_case):
    model = dict(ecstr_case['model'])
    model['alphas_E'] = model['alphas_E'].copy()
    model['alphas_E'][17] = 0.0
    E, F = opredict.Predictor(model).predict(ecstr_case['R'])
    _fails(ecstr_case, E, F, 'force entries')
    _fails(ecstr_case, E, ecstr_case['F'], 'energies')


def test_alphas_E_on_one_permutation_only_fails(ecstr_case):
    """alphas_E of one training point applied to its first permutation instead of all S."""
    sub = opredict.Predictor(ecstr_case['model'])
    S = sub.n_perms
    sub.alphas_E_lin = sub.alphas_E_lin.copy()
    sub.alphas_E_lin[17 * S + 1 : 18 * S] = 0.0
    E, F = sub.predict(ecstr_case['R'])
    _fails(ecstr_case, E, F, 'force entries')
    _fails(ecstr_case, E, ecstr_case['F'], 'energies')


def test_kee_without_cubic_term_fails(ecstr_case):
    """K_ee = (1 + n/sig) e^{-n/sig}: the n/(3 sig) term dropped (the energy alone carries K_ee)."""
    op = ecstr_case['op']
    x, _ = odesc.from_R(ecstr_case['R'])
    n = _norms(op, x)
    dE = -op.std * (op.alphas_E_lin[None] * (n * n / (3 * SIG ** 2)) * np.exp(-n / SIG)).sum(axis=1)
    assert np.all(np.abs(dE) > 0)
    _fails(ecstr_case, ecstr_case['E'] + dE, ecstr_case['F'], 'energies')


def test_kv_energy_rows_with_the_wrong_sign_fail(ecstr_case):
    """K.v on the training points (std = 1, c = 0, R=None) as the iterative solver takes it: energies negated."""
    from sgdml_b200 import synth

    model = dict(ecstr_case['model'], std=1.0, c=0.0)
    x, g = odesc.from_R(synth.geometries(N, M, 0).reshape(M, -1))
    op = opredict.Predictor(model)
    op.set_R_desc(x)
    op.set_R_d_desc(g)
    E, F = op.predict()
    scale = pc.predict_abs_scale(model, oracle=op, R_desc=x, R_d_desc=g)
    k = ecstr_case['k']
    pc.check_predict(E, F, E, F, scale, k)
    with pytest.raises(AssertionError, match='energies'):
        pc.check_predict(-E, F, E, F, scale, k)


# ------------------------------------------------------------------------------------------------ periodic models
def test_pbc_case_wraps(pbc_case):
    lat, lat_inv = pbc_case['op'].lat_and_inv
    _, c = pc._pair_frac(pbc_case['R'], lat_inv)
    assert np.mean(np.any(np.around(c) != 0, axis=-1)) >= 0.2
    x, _ = odesc.from_R(pbc_case['R'], (lat, lat_inv))
    assert np.max(x) <= 1.0  # every image at least 1 A away


def test_lattice_transposed_fails(pbc_case):
    model = dict(pbc_case['model'], lattice=pbc_case['model']['lattice'].T.copy())
    E, F = opredict.Predictor(model).predict(pbc_case['R'])
    _fails(pbc_case, E, F, 'force entries')


def test_one_pair_image_moved_fails(pbc_case):
    """Geometry 21, pair 30: its difference vector moved by the first lattice vector."""
    lat, lat_inv = pbc_case['op'].lat_and_inv
    i, d0 = 21, 30
    R = pbc_case['R'][i : i + 1]
    d, c = pc._pair_frac(R, lat_inv)
    d = d - np.einsum('ij,...j->...i', lat, np.around(c))
    d[0, d0] += lat[:, 0]
    dist = np.sqrt(np.sum(d * d, axis=-1))
    E_i, F_i = _predict_desc(pbc_case['model'], 1 / dist, d / (dist ** 3)[..., None])
    E, F = pbc_case['E'].copy(), pbc_case['F'].copy()
    E[i], F[i] = E_i[0], F_i[0]
    _fails(pbc_case, E, F, 'force entries')


def test_desc_pbc_bound(pbc_case):
    """The descriptor bound passes the np.longdouble evaluation with margin and fails a one-ulp-scale shift of the
    cell."""
    lat, lat_inv = pbc_case['op'].lat_and_inv
    R = pbc_case['R']
    x, g = odesc.from_R(R, (lat, lat_inv))
    xl, gl = _longdouble_desc(R, lat)
    bx, bg = pc.desc_pbc_bound(R, lat, lat_inv)
    assert np.all(np.abs(x - xl) <= bx / 10) and np.all(np.abs(g - gl) <= bg[..., None] / 10)
    x2, g2 = odesc.from_R(R, (lat * (1 + 1e-12), lat_inv))
    assert not np.all(np.abs(g2 - g) <= bg[..., None])


# ------------------------------------------------------------------------------------------------ main-kernel schedule
# dynamic shared memory of k_predict_main per tile class (PCfg::SMEM_BYTES): pinned, so that a change to a class's
# carve-up shows here before the GPU tests' schedules move
SMEM_BYTES = {40: 107552, 72: 193568, 112: 162080, 160: 156192, 224: 205344, 256: 158880}
CLASS_N = {'c1': 12, 'c2': 15, 'c3': 18, 'c4': 21, 'c5': 23}  # one molecule size per persistent tile class


def test_tile_classes_match_the_kernel_source():
    """PCFG is what csrc/predict.cu instantiates (template defaults MINB = 1, W2S = 1, OB = 0), and kCfgs agrees."""
    import os
    import re

    src = open(os.path.join(os.path.dirname(__file__), '..', 'sgdml_b200', 'csrc', 'predict.cu')).read()
    found = {}
    for args in re.findall(r'using Cfg\w+ = PCfg<([\d,\s]+)>;', src):
        a = [int(v) for v in args.split(',')]
        a += [1, 1, 0][len(a) - 8 :]
        found[a[0]] = tuple(a[1:])
    assert found == pc.PCFG
    k = re.search(r'const CfgInfo kCfgs\[\] = \{(.*?)\};', src).group(1)
    assert [tuple(int(v) for v in t) for t in re.findall(r'\{(\d+), (\d+), (\d+)\}', k)] == list(pc._CFGS)


def test_shared_memory_and_residency():
    assert {DP: pc.smem_bytes(DP) for DP in pc.PCFG} == SMEM_BYTES
    assert all(b <= 232448 for b in SMEM_BYTES.values())
    # 152 - 201 KiB: one CTA per SM for every persistent class, two for the D <= 40 class it is compiled for
    assert {DP: pc.ctas_per_sm(DP) for DP in pc.PCFG} == {40: 2, 72: 1, 112: 1, 160: 1, 224: 1, 256: 1}


def test_main_schedule_by_hand():
    # aspirin's first device chunk on 132 SMs: 24 966 x 6 rows in 4 682 tiles of 32; 4 682 = 35 x 132 + 62
    s = pc.main_schedule(21, 1000, 6, 24966, 132)
    assert (s.q_tiles, s.n_tiles, s.n_splits, s.grid, s.per_sm) == (4682, 63, 1, 132, 1)
    assert [len(s.cta_tiles[x]) for x in (0, 61, 62, 131)] == [36, 36, 35, 35]
    assert list(s.cta_tiles[5][:3]) == [5, 137, 269]
    # 37 geometries: ceil(264 / 7) = 38 splits wanted, 2 ceil(sqrt(126)) = 24 allowed, 3 tiles each: 21 pieces; a
    # workspace of just 37 geometries holds one plane of partial sums, so the sweep stays whole
    s = pc.main_schedule(21, 1000, 6, 37, 132)
    assert (s.q_tiles, s.n_splits, s.tiles_per_split, s.grid) == (7, 21, 3, 7)
    s = pc.main_schedule(21, 1000, 6, 37, 132, ws_geo=37)
    assert (s.n_splits, s.grid) == (1, 7)
    # the two-CTA class runs one CTA per query tile
    s = pc.main_schedule(9, 200, 6, 65536, 132)
    assert (s.q_tiles, s.n_splits, s.grid, s.per_sm) == (6144, 1, 6144, 2)
    # class 3, 1 409 geometries: rows 0..31 are geometries 0..5 (5 straddles tiles 0 and 1); tile 264 holds the
    # padded last row block (geometry 1 408, rows 8 448..8 453)
    s = pc.main_schedule(18, 43, 6, 1409, 132)
    assert (s.q_tiles, s.n_tiles, s.grid) == (265, 3, 132)
    assert list(pc.tile_geos(s, 0)) == [0, 1, 2, 3, 4, 5] and list(pc.tile_geos(s, 1)) == list(range(5, 11))
    assert pc.schedule_rows(s, [0]) == [0, 1, 2, 3, 4, 5, 1408]
    assert pc.ragged_round_rows(s) == [1408]
    assert list(pc.straddling_geos(s)[:4]) == [5, 10, 21, 26]


@pytest.mark.parametrize('n_sms', [132, 114])
@pytest.mark.parametrize('cls', sorted(CLASS_N))
def test_multi_sweep_schedules(cls, n_sms):
    """The schedules the persistent-kernel GPU tests run: S = 6, sweeps of 1, 3 and about 8 training tiles (M never a
    multiple of BM), T = 2 grid, 2 grid + 1 and 3 grid - 1 query tiles with the last one padded."""
    N, S = CLASS_N[cls], 6
    BM = pc.layout(N, 100).BM
    for n_tiles, M in ((1, BM - 3), (3, 3 * BM - 5), (8, 8 * BM - 5)):
        grid = pc.main_schedule(N, M, S, 10 ** 6, n_sms).grid
        assert grid == n_sms
        for T, first, last in ((2 * grid, 2, 2), (2 * grid + 1, 3, 2), (3 * grid - 1, 3, 2)):
            B = pc.batch_for_tiles(N, M, S, T)
            s = pc.main_schedule(N, M, S, B, n_sms)
            assert (s.q_tiles, s.n_tiles, s.n_splits, s.grid) == (T, n_tiles, 1, n_sms)
            assert B * S % s.BQ != 0 and -(-(B - 1) * S // s.BQ) < T  # the smallest such batch
            assert len(s.cta_tiles[0]) == first and len(s.cta_tiles[-1]) == last
            assert min(len(t) for t in s.cta_tiles) >= 2
            assert sorted(t for ts in s.cta_tiles for t in ts) == list(range(T))
            # any workspace at least as large as the batch leaves the sweep whole
            assert pc.main_schedule(N, M, S, B, n_sms, ws_geo=B).n_splits == 1
            assert pc.main_schedule(N, M, S, B, n_sms, ws_geo=65536).n_splits == 1
            rr = pc.ragged_round_rows(s)
            n_ragged = T % grid
            assert (len(rr) > 0) == (n_ragged > 0) and (not rr or rr[-1] == B - 1)
            assert not rr or rr[0] == (T - n_ragged) * s.BQ // S
    # one training tile: the sweep is whole even when a few query tiles leave most SMs idle
    s = pc.main_schedule(N, BM - 3, S, 16, n_sms, ws_geo=16)
    assert s.n_splits == 1 and s.grid == s.q_tiles


def test_batch_for_tiles_edges():
    # class 3 (BQ 32), S = 16: 2 geometries fill one tile exactly, so T = 1 needs B = 1 and T = 2 has only B = 3
    assert pc.batch_for_tiles(18, 43, 16, 1) == 1
    assert pc.batch_for_tiles(18, 43, 16, 2) == 3
    # S = 32: every batch fills its tiles exactly
    with pytest.raises(ValueError):
        pc.batch_for_tiles(18, 43, 32, 5)


# ------------------------------------------------------------------------------------------------ schedule faults
# A class 3 shape (D = 153, BQ 32, BM 16) with a sweep of three training tiles (M = 43, the last tile 11 points) and
# T = 2 grid + 1 query tiles at 132 SMs; query tile t = grid + 7 is the second sweep of CTA 7, and its geometries that
# lie wholly inside it get the outputs a schedule fault would give all their rows.  The virtual row (b, p) of the
# kernel pairs with the oracle's permuted cache rows m S + p (m = 0..M-1).
FN, FM, FS, F_SMS = 18, 43, 6, 132


@pytest.fixture(scope='module')
def fault_case():
    from test_predict_ecstr_pbc import _make, _queries

    model, _, _ = _make(FN, FM, seed=FN, ecstr=True)
    B = pc.batch_for_tiles(FN, FM, FS, 2 * F_SMS + 1)
    s = pc.main_schedule(FN, FM, FS, B, F_SMS)
    assert (s.n_tiles, s.n_splits, s.grid, s.BQ) == (3, 1, F_SMS, 32) and s.grid * s.BQ % FS == 0
    t = s.grid + 7
    geos = [b for b in pc.tile_geos(s, t) if b * FS // s.BQ == t == ((b + 1) * FS - 1) // s.BQ]
    assert len(geos) >= 4
    R = _queries(FN, B, 77)
    op = opredict.Predictor(model)
    E, F = op.predict(R[geos])
    k = pc.n_terms(FM, FS, FN * (FN - 1) // 2)
    scale = pc.predict_abs_scale(model, R[geos], oracle=op)
    fc = dict(model=model, op=op, R=R, geos=geos, sched=s, E=E, F=F, k=k, scale=scale)
    E0, F0 = _fault_predict(fc)  # no fault: the construction itself passes
    pc.check_predict(E0, F0, E, F, scale, k)
    return fc


def _fault_predict(fc, keep=None, extra=None, ae=None, src=None):
    """Oracle outputs of the fault case's geometries with the cache rows `keep` (then the rows `extra` once more),
    alphas_E per cache row `ae`, or the query descriptors of geometries `src` under each geometry's own Jacobian."""
    op = fc['op']
    sub = opredict.Predictor(fc['model'])
    idx = np.arange(op.R_desc_perms.shape[0]) if keep is None else keep
    if extra is not None:
        idx = np.concatenate([idx, extra])
    sub.R_desc_perms = op.R_desc_perms[idx]
    sub.R_d_desc_alpha_perms = op.R_d_desc_alpha_perms[idx]
    sub.alphas_E_lin = (op.alphas_E_lin if ae is None else ae)[idx]
    geos = fc['geos']
    x, g = odesc.from_R(fc['R'][geos])
    if src is not None:
        x, _ = odesc.from_R(fc['R'][src])
    E = np.array([sub._raw(xi, gi) for xi, gi in zip(x, g)])
    return E[:, 0] * op.std + op.c, E[:, 1:] * op.std


def _tile_cache_rows(j):
    """The oracle's cache rows m S + p of training tile j (all S permutations)."""
    BM = pc.layout(FN, FM).BM
    m = np.arange(j * BM, min((j + 1) * BM, FM))
    return (m[:, None] * FS + np.arange(FS)[None]).ravel()


def _rejects(fc, E, F):
    assert not np.array_equal(F, fc['F'])
    with pytest.raises(AssertionError, match='force entries'):
        pc.check_predict(E, F, fc['E'], fc['F'], fc['scale'], fc['k'])
    with pytest.raises(AssertionError, match='energies'):
        pc.check_predict(E, fc['F'], fc['E'], fc['F'], fc['scale'], fc['k'])


def test_schedule_fault_dropped_training_tile_fails(fault_case):
    n = FM * FS
    for j in range(3):
        _rejects(fault_case, *_fault_predict(fault_case, keep=np.setdiff1d(np.arange(n), _tile_cache_rows(j))))


def test_schedule_fault_training_tile_twice_fails(fault_case):
    for j in range(3):
        _rejects(fault_case, *_fault_predict(fault_case, extra=_tile_cache_rows(j)))


def test_schedule_fault_previous_sweeps_query_tile_fails(fault_case):
    """Tile t - grid's Q rows in place of tile t's: grid BQ rows back is grid BQ / S whole geometries back, with the
    same permutation in each row."""
    s = fault_case['sched']
    shift = s.grid * s.BQ // FS
    _rejects(fault_case, *_fault_predict(fault_case, src=[b - shift for b in fault_case['geos']]))


def test_schedule_fault_neighbouring_alphas_E_fails(fault_case):
    """Training tile 0 paired with the alphas_E of tile 1 (the aes stage of the other pipeline stage)."""
    op = fault_case['op']
    ae = op.alphas_E_lin.copy()
    ae[_tile_cache_rows(0)] = op.alphas_E_lin[_tile_cache_rows(1)]
    _rejects(fault_case, *_fault_predict(fault_case, ae=ae))
