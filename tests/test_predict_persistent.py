"""The persistent main kernel of the predictor (k_predict_main, csrc/predict.cu) with two and more query tiles per CTA,
in every persistent tile class, against the oracle and bit for bit across schedules.

A CTA of the persistent kernel runs query tiles x, x + grid, ...; the model tiles stream through two shared-memory
stages without a break between sweeps, one running counter sets each tile's stage and mbarrier parity, and the warps
build each Q tile themselves (or, on the zero-copy graph path, wait for it on a third mbarrier).  A slip there gives
some rows a wrong model tile or a stale Q tile and nothing else, so every case here is chosen by
predict_checks.main_schedule to give every CTA at least two sweeps: sweeps of one training tile (each reloads the same
tile into the other stage), of three (odd: a tile changes stage from one sweep to the next) and of about eight, with
T = 2 grid, 2 grid + 1 (CTA 0 alone runs a third sweep) and 3 grid - 1 query tiles (a ragged last round), the last
tile partly padded.  The checked rows are the first and last query tile of CTAs 0, 1 and grid - 1, the ragged round,
the padded tile, geometries whose rows straddle two tiles and a seeded sample, each within the bound of
tests/predict_checks.py with a 10x margin.  Every case prints its schedule."""

import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import predict_checks as pc  # noqa: E402
from conftest import rel_err  # noqa: E402
from oracle import assemble as oassemble  # noqa: E402
from oracle import predict as opredict  # noqa: E402
from test_predict_bulk import _check, _chunk_cap, _main_launches, _model, _nan_out, _plan, _run  # noqa: E402
from test_predict_ecstr_pbc import _env, _make, _queries, _raw_oracle  # noqa: E402

CLASSES = {'c1': 12, 'c2': 15, 'c3': 18, 'c4': 21, 'c5': 23}  # D = 66, 105, 153, 210, 253
S = 6  # the permutation group of _make: one rotor, one swap


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


@pytest.fixture(scope='module')
def n_sms(eng):
    import torch

    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _sweep_M(N, n_tiles):
    """M for a sweep of n_tiles training tiles, never a multiple of BM."""
    BM = pc.layout(N, 100).BM
    return {1: BM - 3, 3: 3 * BM - 5, 8: 8 * BM - 5}[n_tiles]


def _describe(tag, s):
    n = [len(t) for t in s.cta_tiles]
    print('\n[schedule] %s: B %d, q_tiles %d, n_splits %d, grid %d (%d per SM), query tiles per CTA %d..%d (CTA 0: %d), '
          'sweep %d training tiles' % (tag, s.B, s.q_tiles, s.n_splits, s.grid, s.per_sm, min(n), max(n), n[0], s.n_tiles))


def _multi_sweep(tag, s, third_on_cta0=False):
    _describe(tag, s)
    n = [len(t) for t in s.cta_tiles]
    assert s.n_splits == 1 and min(n) >= 2, 'not a multi-sweep schedule'
    if third_on_cta0:
        assert n[0] == 3 and n[1:] == [2] * (s.grid - 1)


def _schedule_rows(s, seed):
    """The rows a schedule fault would show in: first and last query tile of CTAs 0, 1 and grid - 1, the ragged round,
    the padded last tile, 16 straddling geometries and 32 seeded ones."""
    rng = np.random.default_rng(seed)
    rows = set(pc.schedule_rows(s, (0, 1, s.grid - 1)))
    rows.update(pc.ragged_round_rows(s))
    rows.update(pc.tile_geos(s, s.q_tiles - 1))
    st = pc.straddling_geos(s)
    rows.update(int(b) for b in rng.choice(st, size=min(16, len(st)), replace=False))
    rows.update(int(b) for b in rng.choice(s.B, size=min(32, s.B), replace=False))
    return sorted(rows)


def _np(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


# --------------------------------------------------------------------------- a. every class, every sweep length
@pytest.mark.parametrize('n_tiles', [1, 3, 8])
@pytest.mark.parametrize('cls', sorted(CLASSES))
def test_every_class_multi_sweep(eng, n_sms, cls, n_tiles):
    """Device tensors at T = 2 grid, 2 grid + 1 and 3 grid - 1 query tiles, one launch each; with a sweep of three
    tiles also pageable NumPy arrays of four chunks of 2 grid + 1 tiles each, pipelined on the two workspace slots."""
    import torch

    N = CLASSES[cls]
    M = _sweep_M(N, n_tiles)
    model, _, _ = _make(N, M, seed=N + n_tiles, ecstr=False)
    op = opredict.Predictor(model)
    p = eng.GDMLPredict(model)
    grid = pc.main_schedule(N, M, S, 10 ** 6, n_sms).grid
    assert grid == n_sms
    for T in (2 * grid, 2 * grid + 1, 3 * grid - 1):
        B = pc.batch_for_tiles(N, M, S, T)
        s = pc.main_schedule(N, M, S, B, n_sms)
        tag = '%s sweep %d T %d' % (cls, n_tiles, T)
        _multi_sweep(tag, s, third_on_cta0=T == 2 * grid + 1)
        assert s.n_tiles == n_tiles and s.q_tiles == T
        R = _queries(N, B, 1000 * n_tiles + T)
        plan = _plan(model, B, False)
        assert plan.main_launches == 1
        E, F = _run(p, torch.from_numpy(R).cuda(), plan)
        _check(tag, model, op, R, _schedule_rows(s, T), _np(E), _np(F))
    if n_tiles != 3:
        return
    c = pc.batch_for_tiles(N, M, S, 2 * grid + 1)
    B = 4 * c
    plan = _plan(model, B, True)
    assert plan.pipelined and plan.slots == [0, 1, 0, 1] and plan.chunks == [(i * c, (i + 1) * c) for i in range(4)]
    s = pc.main_schedule(N, M, S, c, n_sms)
    _multi_sweep('%s sweep 3 host, 4 chunks of' % cls, s, third_on_cta0=True)
    R = _queries(N, B, 77 + N)
    E, F = _run(p, R, plan, out=_nan_out(B, 3 * N, numpy=True))
    rows = [lo + r for lo, _ in plan.chunks for r in pc.schedule_rows(s, (0, 1, s.grid - 1)) + pc.ragged_round_rows(s)]
    _check('%s sweep 3 host B=%d' % (cls, B), model, op, R, rows, E, F)


# --------------------------------------------------------------------------- b. bit for bit across schedules
def _cap_for(N, M, S_, n_sms):
    """The smallest chunk cap that keeps every tile's rows (cap S = 0 mod BQ) and a whole sweep (at least 2 n_sms
    tiles), with a tile count that is no multiple of n_sms, so that the capped chunks put each tile on another CTA."""
    BQ = pc.layout(N, M).BQ
    step = BQ // math.gcd(S_, BQ)
    cap = step
    while cap * S_ // BQ < 2 * n_sms or (cap * S_ // BQ) % n_sms == 0:
        cap += step
    return cap


def _across_schedules(eng, model, N, M, S_, n_sms, R, cap, tag):
    import torch

    B = R.shape[0]
    Rd = torch.from_numpy(R).cuda()
    p = eng.GDMLPredict(model)
    s = pc.main_schedule(N, M, S_, B, n_sms)
    _describe('%s uncapped' % tag, s)
    E1, F1 = _run(p, Rd, _plan(model, B, False))
    E1, F1 = _np(E1), _np(F1)
    with _chunk_cap(cap):
        q = eng.GDMLPredict(model)
        plan = _plan(model, B, False, cap=cap)
        for lo, hi in plan.chunks:
            sc = pc.main_schedule(N, M, S_, hi - lo, n_sms)
            _describe('%s chunk [%d, %d)' % (tag, lo, hi), sc)
            assert sc.n_splits == 1
        assert len(plan.chunks) >= 2
        E2, F2 = _run(q, Rd, plan)
    assert np.array_equal(_np(E2), E1) and np.array_equal(_np(F2), F1), '%s: the capped schedule differs' % tag


@pytest.mark.parametrize('cls', ['c0'] + sorted(CLASSES))
def test_bit_identical_across_schedules(eng, n_sms, cls):
    """A batch in one launch and in chunks of `cap` geometries: the same rows in every tile, but on other CTAs and in
    other sweeps, so E and F agree bit for bit.  c0 (D <= 40, one CTA per query tile) is the control."""
    N = 9 if cls == 'c0' else CLASSES[cls]
    M = _sweep_M(N, 3) if cls != 'c0' else 3 * 32 - 5
    model, _, _ = _make(N, M, seed=50 + N, ecstr=False)
    cap = _cap_for(N, M, S, n_sms)
    r = pc.batch_for_tiles(N, M, S, 2 * n_sms)
    assert r < cap
    R = _queries(N, 2 * cap + r, 60 + N)
    _across_schedules(eng, model, N, M, S, n_sms, R, cap, '%s cap %d' % (cls, cap))
    if cls == 'c4':
        from sgdml_b200 import synth

        perms, r0 = synth.config_perms_and_r0('aspirin')
        Ma = 1000
        am, _, _ = _model(21, Ma, perms, 20, r0=r0)
        Sa = len(perms)
        cap = _cap_for(21, Ma, Sa, n_sms)
        B = 3 * cap + pc.batch_for_tiles(21, Ma, Sa, 2 * n_sms + 1)
        Ra = synth.geometries(21, B, 5, r0=r0).reshape(B, -1)
        _across_schedules(eng, am, 21, Ma, Sa, n_sms, Ra, cap, 'aspirin M=1000 cap %d' % cap)


# --------------------------------------------------------------------------- c. energy constraints and cells
@pytest.mark.parametrize('kind', ['ecstr', 'pbc'])
@pytest.mark.parametrize('cls', ['c2', 'c3', 'c5'])
def test_energy_constraints_and_cells_multi_sweep(eng, n_sms, cls, kind):
    """alphas_E (the aes stage of every model tile) or a fixed skewed cell, sweeps of three tiles, T = 2 grid + 1."""
    import torch

    N = CLASSES[cls]
    M = _sweep_M(N, 3)
    lat = pc.skewed_cell(N) if kind == 'pbc' else None
    model, _, _ = _make(N, M, seed=70 + N, ecstr=kind == 'ecstr', lattice=lat)
    op = opredict.Predictor(model)
    B = pc.batch_for_tiles(N, M, S, 2 * n_sms + 1)
    s = pc.main_schedule(N, M, S, B, n_sms)
    tag = '%s %s sweep 3 T %d' % (kind, cls, s.q_tiles)
    _multi_sweep(tag, s, third_on_cta0=True)
    R = _queries(N, B, 80 + N, lat)
    p = eng.GDMLPredict(model)
    E, F = _run(p, torch.from_numpy(R).cuda(), _plan(model, B, False))
    _check(tag, model, op, R, _schedule_rows(s, 3), _np(E), _np(F))


# --------------------------------------------------------------------------- d. zero-copy graph path
@pytest.mark.parametrize('N,rotors,swaps', [(18, 3, 4), (21, 4, 4)])
def test_graph_zero_copy_multi_sweep(eng, n_sms, monkeypatch, N, rotors, swaps):
    """16 host geometries replayed from a captured graph whose main kernel waits for each prepared Q tile on its
    third mbarrier: S = 432 (216 tiles) and S = 1296 (648 tiles), one training tile (no split).  Every row against the
    oracle, and bit-identical to the graph that builds Q in the kernel and to the path without a graph."""
    from sgdml_b200 import synth

    perms = synth.rotor_swap_group(N, rotors, swaps)
    S_ = len(perms)
    M = pc.layout(N, 100).BM - 3
    model, _, _ = _model(N, M, perms, 20, seed=N)
    B = 16
    s = pc.main_schedule(N, M, S_, B, n_sms)
    _describe('graph N=%d S=%d' % (N, S_), s)
    assert s.n_splits == 1 and s.q_tiles > s.grid and len(s.cta_tiles[0]) >= 2
    R_cap, R = _queries(N, B, 90 + N), _queries(N, B, 91 + N)
    with _env(monkeypatch, SGDML_B200_GRAPH='1', SGDML_B200_GRAPH_ZEROCOPY='1'):
        pg = eng.GDMLPredict(model)
        pg.predict(R_cap)  # captures
        E, F = _run(pg, R, _plan(model, B, True), out=_nan_out(B, 3 * N, numpy=True))  # replays
    _check('graph zero copy N=%d S=%d' % (N, S_), model, opredict.Predictor(model), R, range(B), E, F)
    for env in ({'SGDML_B200_GRAPH': '1', 'SGDML_B200_GRAPH_ZEROCOPY': '0'}, {'SGDML_B200_GRAPH': '0'}):
        with _env(monkeypatch, **env):
            q = eng.GDMLPredict(model)
            q.predict(R_cap)
            E2, F2 = q.predict(R)
        assert np.array_equal(E2, E) and np.array_equal(F2, F), 'zero-copy replay differs from %s' % env


# --------------------------------------------------------------------------- e. K.v over long training ranges
KV_CLASSES = ('c2', 'c3', 'c4')
KV_PERMS = (2, 2)  # rotors, swaps: S = 36


def _kv_case(eng, n_sms, cls, seed):
    """A model of M = L + 48 training points, L = ceil(2 n_sms BQ / S) so that a range of L points is 2 n_sms query
    tiles; the three ranges start at 0, at 37 and end at M, and all contain the points 48..L-1."""
    from sgdml_b200 import synth

    N = CLASSES[cls]
    perms = synth.rotor_swap_group(N, *KV_PERMS)
    S_ = len(perms)
    BQ = pc.layout(N, 100).BQ
    L = -(-2 * n_sms * BQ // S_)
    M = L + 48
    model, x, g = _model(N, M, perms, 20, seed=seed)
    ranges = [(0, L), (37, 37 + L), (M - L, M)]
    for lo, hi in ranges + [(0, M)]:
        s = pc.main_schedule(N, M, S_, hi - lo, n_sms)
        _describe('%s K.v [%d, %d)' % (cls, lo, hi), s)
        assert s.n_splits == 1 and min(len(t) for t in s.cta_tiles) >= 2
    rng = np.random.default_rng(seed)
    pts = sorted(set(rng.choice(np.arange(M - L, L), size=24, replace=False).tolist())
                 | {r for lo, hi in ranges for r in (lo, hi - 1)})
    p = eng.GDMLPredict(model)
    p.set_R_desc(x)
    p.set_R_d_desc(g)
    return N, M, S_, BQ, model, x, g, ranges, pts, p


def _kv(p, lo, hi, dim_i, with_E):
    F = np.full((hi - lo, dim_i), np.nan)
    E = np.full(hi - lo, np.nan) if with_E else None
    n0 = _main_launches()
    p.kmatvec_train(lo, hi, out=F, E_out=E)
    assert _main_launches() - n0 == 1
    return E, F


def _aligned_subranges(p, M, S_, BQ, ranges, full, dim_i, with_E):
    """[0, L) and [a, M), a the largest multiple of BQ / gcd(BQ, S) <= M - L: the same rows in every query tile as in
    the full range, on other CTAs and in other sweeps -- bit for bit."""
    step = BQ // math.gcd(BQ, S_)
    a = (ranges[2][0] // step) * step
    assert a > 0 and a * S_ % BQ == 0
    for lo, hi in ((0, ranges[0][1]), (a, M)):
        E, F = _kv(p, lo, hi, dim_i, with_E)
        assert np.array_equal(F, full[1][lo:hi]), 'K.v [%d, %d) differs from the full range' % (lo, hi)
        if with_E:
            assert np.array_equal(E, full[0][lo:hi])


@pytest.mark.parametrize('cls', ['c2', 'c4'])
def test_kv_long_ranges(eng, n_sms, cls):
    """K.v = kmatvec_train over ranges of 2 n_sms query tiles: 30 sampled training points against the oracle's kernel
    matrix columns (K is symmetric: row block j of K v is column block j of K, transposed, times v)."""
    N, M, S_, BQ, model, x, g, ranges, pts, p = _kv_case(eng, n_sms, cls, seed=110 + CLASSES[cls])
    dim_i = 3 * N
    v = np.random.default_rng(5).standard_normal(M * dim_i)
    p.set_alphas(v)
    lin = model['tril_perms_lin']
    ref = {j: oassemble.assemble(x, g, lin, 20, col_idxs=np.arange(j * dim_i, (j + 1) * dim_i)).T @ v for j in pts}
    for lo, hi in ranges:
        _, F = _kv(p, lo, hi, dim_i, False)
        js = [j for j in pts if lo <= j < hi]
        err = rel_err(np.stack([F[j - lo] for j in js]), np.stack([ref[j] for j in js]))
        print('\n[K.v] %s [%d, %d): %d points, rel_err %.2e' % (cls, lo, hi, len(js), err))
        assert len(js) >= 26 and err < 1e-10
    full = _kv(p, 0, M, dim_i, False)
    _aligned_subranges(p, M, S_, BQ, ranges, full, dim_i, False)


def test_kv_long_ranges_energy_constraints(eng, n_sms):
    """c3 with alphas_E: force rows and raw energy sums (E_out) of 30 sampled training points against the oracle
    predictor on those points (std = 1, c = 0), within the bound with a 10x margin."""
    N, M, S_, BQ, model, x, g, ranges, pts, p = _kv_case(eng, n_sms, 'c3', seed=130)
    dim_i = 3 * N
    rng = np.random.default_rng(6)
    vF, vE = rng.standard_normal(M * dim_i), rng.standard_normal(M)
    p.set_alphas(vF, alphas_E=vE)
    m, op = _raw_oracle(model, x, g, vF, vE)
    op.set_R_desc(x[pts])
    op.set_R_d_desc(g[pts])
    E_ref, F_ref = op.predict()
    scale = pc.predict_abs_scale(m, oracle=op, R_desc=x[pts], R_d_desc=g[pts])
    k = pc.n_terms(M, S_, x.shape[1])
    pos = {j: i for i, j in enumerate(pts)}
    for lo, hi in ranges:
        E, F = _kv(p, lo, hi, dim_i, True)
        js = [j for j in pts if lo <= j < hi]
        sel = [pos[j] for j in js]
        rF, rE = pc.check_predict(E[np.array(js) - lo], F[np.array(js) - lo], E_ref[sel], F_ref[sel],
                                  (scale[0][sel], scale[1][sel]), k, what='c3 ecstr K.v [%d, %d)' % (lo, hi))
        print('\n[predict bound] c3 ecstr K.v [%d, %d): %d points, max|err|/scale F %.2e E %.2e, tau %.2e'
              % (lo, hi, len(js), rF, rE, pc.tau(k)))
        assert len(js) >= 26 and rF <= pc.tau(k) / 10 and rE <= pc.tau(k) / 10
    full = _kv(p, 0, M, dim_i, True)
    _aligned_subranges(p, M, S_, BQ, ranges, full, dim_i, True)
