"""Energy-constrained and periodic models in every predictor tile class against the oracle.

Energy constraints in the kernel (alphas_E, use_E_cstr models) run the matern52_ecstr branches of the main kernel: the
fused register transform of D <= 112, the split-k row-half exchange of the BQ 32 x BM 16 classes (D <= 224), the
shared-memory split-k transform of 224 < D <= 256 and the GEMM-composed path of D > 256.  Periodic models build
their query descriptors with the minimum-image convention in two kernels, k_desc_from_R (chunked path, device
tensors, copy-node graph) and k_desc_query_rows (zero-copy graph), which must pick the same images -- also at exact
rounding ties -- and round alike.  Captured graphs carry use_ae as a kernel argument, so set_alphas_E must invalidate
them; they read the cell staged by each call, so after set_lattice a replay must see the new cell; and a rejected
set_lattice must leave the model as it was.

Every model is built with the oracle's descriptor code.  Output buffers passed with out= are filled with NaN first,
and two calls on one handle see different inputs.  Each check prints max |err| / scale against tau (10x margin)."""

import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import predict_checks as pc  # noqa: E402
from conftest import rel_err  # noqa: E402
from ecstr_oracle import kernel_op_ecstr  # noqa: E402
from oracle import assemble as oassemble  # noqa: E402
from oracle import desc as odesc  # noqa: E402
from oracle import predict as opredict  # noqa: E402
from oracle import train as otrain  # noqa: E402
from test_predict_bulk import _chunk_cap, _check, _nan_out, _plan, _run  # noqa: E402

ERR_ARG = -1000
SIG = 20
# name: (N, M, DP or None for the GEMM-composed path); M is never a multiple of BM and spans at least three tiles
SHAPES = {
    'c0': (9, 70, 40),
    'c1': (12, 70, 72),
    'c2': (15, 41, 112),
    'c3': (18, 41, 160),
    'c4': (21, 41, 224),
    'c5': (23, 29, 256),
    'large': (24, 19, None),
}
PBC_SHAPES = ('c0', 'c3', 'c4', 'c5', 'large')
MARGIN = 1e-6


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


def _lat_inv(lat):
    return np.ascontiguousarray(np.linalg.inv(lat))


def _make(N, M, seed, ecstr, lattice=None):
    """Random-coefficient model (std and c away from 1 and 0); with ecstr, seeded mixed-sign alphas_E large enough to
    move E and F by well over 10 %; with a lattice, training descriptors in that cell.  Returns (model, x, g)."""
    from sgdml_b200 import synth

    perms = synth.rotor_swap_group(N, 1, 1)
    R = synth.geometries(N, M, seed).reshape(M, -1)
    rng = np.random.default_rng(seed + 99)
    alphas = rng.standard_normal(M * 3 * N)
    x, g = odesc.from_R(R, None if lattice is None else (lattice, _lat_inv(lattice)))
    model = {
        'type': 'm',
        'z': np.ones(N, dtype=np.int64),
        'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(g, alphas.reshape(M, -1)),
        'alphas_F': alphas,
        'c': 0.37,
        'std': 1.7,
        'sig': SIG,
        'lam': 1e-10,
        'perms': perms,
        'tril_perms_lin': odesc.tril_perms_lin(perms),
        'use_E': True,
    }
    if ecstr:
        model['alphas_E'] = 3.0 * rng.standard_normal(M)
    if lattice is not None:
        model['lattice'] = lattice
    return model, x, g


def _queries(N, B, seed, lattice=None):
    """B seeded query geometries; in a cell, those within MARGIN of a rounding tie are replaced (few are)."""
    from sgdml_b200 import synth

    if lattice is None:
        return synth.geometries(N, B, seed).reshape(B, -1)
    R = synth.geometries(N, 2 * B, seed).reshape(2 * B, -1)
    keep = pc.pbc_margin(R, lattice, _lat_inv(lattice)) >= MARGIN
    assert np.sum(~keep[:B]) <= max(2, B // 20), 'too many queries near a rounding tie'
    return np.ascontiguousarray(R[keep][:B])


def _assert_layout(N, M, DP):
    ly = pc.layout(N, M)
    assert ly.large == (DP is None) and (DP is None or ly.DP == DP)
    assert M % ly.BM != 0 and ly.Mpad // ly.BM >= 3


@contextlib.contextmanager
def _env(monkeypatch, **kv):
    with monkeypatch.context() as mp:
        for k, v in kv.items():
            mp.setenv(k, v)
        yield


def _torch():
    import torch

    return torch


def _routes(eng, model, op, N, Rs, monkeypatch, tag):
    """The routes of one model against the oracle.  Rs: dict of query batches (different inputs per call)."""
    torch = _torch()
    dim_i = 3 * N
    # host batch of 37 (chunked path, NaN-filled out=)
    p = eng.GDMLPredict(model)
    out = _nan_out(37, dim_i, numpy=True)
    E, F = _run(p, Rs['h37'], _plan(model, 37, True), out=out)
    _check('%s host B=37' % tag, model, op, Rs['h37'], range(37), E, F)
    # CUDA tensors: B = 1 (the sweep over M split across CTAs) and B = 37
    for key in ('d1', 'd37'):
        R = Rs[key]
        E, F = _run(p, torch.from_numpy(R).cuda(), _plan(model, R.shape[0], False))
        _check('%s device B=%d' % (tag, R.shape[0]), model, op, R, range(R.shape[0]), E, F)
    # at most 5 queries per chunk: 8 chunks
    with _chunk_cap(5):
        pc5 = eng.GDMLPredict(model)
        plan = _plan(model, 37, True, cap=5)
        assert len(plan.chunks) == 8
        out = _nan_out(37, dim_i, numpy=True)
        E, F = _run(pc5, Rs['cap'], plan, out=out)
    _check('%s host B=37 cap 5' % tag, model, op, Rs['cap'], range(37), E, F)
    # B = 3 through the graph, zero-copy and copy-node forms (one handle each: the graph cache does not key on the
    # form), bit-identical to the chunked path of the same call
    R3 = Rs['g3']
    with _env(monkeypatch, SGDML_B200_GRAPH='0'):
        E0, F0 = eng.GDMLPredict(model).predict(R3)
    _check('%s host B=3 chunked' % tag, model, op, R3, range(3), E0, F0)
    for zc in ('1', '0'):
        with _env(monkeypatch, SGDML_B200_GRAPH='1', SGDML_B200_GRAPH_ZEROCOPY=zc):
            pg = eng.GDMLPredict(model)
            pg.predict(Rs['h37'][:3])  # captures the graph
            out = _nan_out(3, dim_i, numpy=True)
            E, F = _run(pg, R3, _plan(model, 3, True), out=out)  # replays it
        assert np.array_equal(E, E0) and np.array_equal(F, F0), 'graph (zero copy %s) differs from the chunked path' % zc
    return p


def _batches(N, seed, lattice=None):
    return {
        'h37': _queries(N, 37, seed, lattice),
        'd1': _queries(N, 1, seed + 1, lattice),
        'd37': _queries(N, 37, seed + 2, lattice),
        'cap': _queries(N, 37, seed + 3, lattice),
        'g3': _queries(N, 3, seed + 4, lattice),
    }


def _training_points(eng, p, model, op, x, g, tag):
    """predict() on the training points: the self-terms, n = 0 and K_ee = 1."""
    p.set_R_desc(x)
    p.set_R_d_desc(g)
    E, F = p.predict()
    op.set_R_desc(x)
    op.set_R_d_desc(g)
    E_ref, F_ref = op.predict()
    M, D = x.shape
    k = pc.n_terms(M, op.n_perms, D)
    scale = pc.predict_abs_scale(model, oracle=op, R_desc=x, R_d_desc=g)
    rF, rE = pc.check_predict(E, F, E_ref, F_ref, scale, k, what='%s R=None' % tag)
    print('\n[predict bound] %s R=None: max|err|/scale F %.2e E %.2e, tau %.2e' % (tag, rF, rE, pc.tau(k)))
    assert rF <= pc.tau(k) / 10 and rE <= pc.tau(k) / 10


def _raw_oracle(model, x, g, vF, vE):
    """Oracle predictor of the raw K.v sums (std = 1, c = 0) for alphas = [vF; vE] on the training points."""
    M = x.shape[0]
    m = dict(model, std=1.0, c=0.0, R_d_desc_alpha=odesc.d_desc_dot_vec(g, vF.reshape(M, -1)))
    if vE is None:
        m.pop('alphas_E', None)
    else:
        m['alphas_E'] = vE
    op = opredict.Predictor(m)
    op.set_R_desc(x)
    op.set_R_d_desc(g)
    return m, op


def _check_kv(p, model, x, g, vF, vE, ranges, tag, K_full=None):
    """kmatvec_train with E_out over [lo, hi) against the oracle's raw sums, within the bound at std = 1; with K_full,
    also against K_full @ v (the explicit energy-constrained matrix: K v = [F; -E])."""
    M, D = x.shape
    dim_i = 3 * odesc.n_atoms_from_dim(D)
    m, op = _raw_oracle(model, x, g, vF, vE)
    E_ref, F_ref = op.predict()
    scale = pc.predict_abs_scale(m, oracle=op, R_desc=x, R_d_desc=g)
    k = pc.n_terms(M, op.n_perms, D)
    worst = 0.0
    for lo, hi in ranges:
        F = np.full((hi - lo, dim_i), np.nan)
        E = np.full(hi - lo, np.nan) if vE is not None else None
        p.kmatvec_train(lo, hi, out=F, E_out=E)
        sl = slice(lo, hi)
        rF, rE = pc.check_predict(E, F, None if E is None else E_ref[sl], F_ref[sl], (scale[0][sl], scale[1][sl]), k,
                                  what='%s K.v [%d, %d)' % (tag, lo, hi))
        worst = max(worst, rF, rE or 0.0)
        if K_full is not None:
            Kv = K_full @ np.concatenate([vF, vE])
            assert rel_err(F.ravel(), Kv[lo * dim_i : hi * dim_i]) < 1e-10
            assert rel_err(-E, Kv[M * dim_i + lo : M * dim_i + hi]) < 1e-10
    print('\n[predict bound] %s K.v: max|err|/scale %.2e, tau %.2e' % (tag, worst, pc.tau(k)))
    assert worst <= pc.tau(k) / 10
    return E_ref, F_ref


# --------------------------------------------------------------------------- 2. energy constraints, every class
@pytest.mark.parametrize('name', sorted(SHAPES))
def test_energy_constraints_every_tile_class(eng, monkeypatch, name):
    N, M, DP = SHAPES[name]
    _assert_layout(N, M, DP)
    model, x, g = _make(N, M, seed=N, ecstr=True)
    op = opredict.Predictor(model)
    Rs = _batches(N, 100 + N)
    # alphas_E matters: without it E and F move by at least 10 % of their largest entry
    E1, F1 = op.predict(Rs['h37'])
    m0 = dict(model)
    del m0['alphas_E']
    E0, F0 = opredict.Predictor(m0).predict(Rs['h37'])
    assert np.max(np.abs(E1 - E0)) >= 0.1 * np.max(np.abs(E1))
    assert np.max(np.abs(F1 - F0)) >= 0.1 * np.max(np.abs(F1))

    p = _routes(eng, model, op, N, Rs, monkeypatch, 'ecstr %s' % name)
    _training_points(eng, p, model, op, x, g, 'ecstr %s' % name)

    # K.v with energy rows: v = [v_F; v_E] against the oracle's operator and the explicit matrix
    rng = np.random.default_rng(7 + N)
    vF, vE = rng.standard_normal(M * 3 * N), rng.standard_normal(M)
    p.set_alphas(vF, alphas_E=vE)
    ranges = [(0, M), (5, M - 7), (M - 1, M)]
    K = oassemble.assemble_E_cstr(x, g, model['tril_perms_lin'], SIG)
    E_ref, F_ref = _check_kv(p, model, x, g, vF, vE, ranges, 'ecstr %s' % name, K_full=K)
    Kop = kernel_op_ecstr(model, x, g, 0.0)(np.concatenate([vF, vE]))
    assert rel_err(Kop, np.concatenate([F_ref.ravel(), -E_ref])) < 1e-12


# --------------------------------------------------------------------------- 3. periodic models
@pytest.mark.parametrize('name', PBC_SHAPES)
def test_periodic_every_route(eng, monkeypatch, name):
    """(a) the skewed cell wraps, (b) every route against the oracle with model['lattice'], graph routes bit-identical
    to the chunked route, (d) moving query atoms by lattice vectors stays within the bound."""
    N, M, DP = SHAPES[name]
    _assert_layout(N, M, DP)
    lat = pc.skewed_cell(N)
    lat_inv = _lat_inv(lat)
    model, x, g = _make(N, M, seed=N + 1, ecstr=False, lattice=lat)
    op = opredict.Predictor(model)
    Rs = _batches(N, 200 + N, lat)
    R = Rs['h37']
    _, c = pc._pair_frac(R, lat_inv)
    assert np.mean(np.any(np.around(c) != 0, axis=-1)) >= 0.2, 'fewer than 20 % of the pairs wrap'
    xq, _ = odesc.from_R(R, (lat, lat_inv))
    assert np.max(xq) <= 1.0, 'an image closer than 1 A'
    assert np.min(pc.pbc_margin(R, lat, lat_inv)) >= MARGIN

    p = _routes(eng, model, op, N, Rs, monkeypatch, 'pbc %s' % name)
    _training_points(eng, p, model, op, x, g, 'pbc %s' % name)

    # (d) integer combinations of lattice vectors added to random atoms: the same images, so the same E and F
    rng = np.random.default_rng(N)
    n = rng.integers(-1, 2, size=(R.shape[0], N, 3)) * (rng.random((R.shape[0], N, 1)) < 0.5)
    Rsh = (R.reshape(-1, N, 3) + np.einsum('ij,bnj->bni', lat, n)).reshape(R.shape)
    assert np.any(Rsh != R)
    E, F = p.predict(Rsh)
    E_ref, F_ref = op.predict(R)
    k = pc.n_terms(M, op.n_perms, N * (N - 1) // 2)
    rF, rE = pc.check_predict(E, F, E_ref, F_ref, pc.predict_abs_scale(model, R, oracle=op), k, what='pbc %s shifted' % name)
    print('\n[predict bound] pbc %s atoms moved by lattice vectors: max|err|/scale F %.2e E %.2e, tau %.2e'
          % (name, rF, rE, pc.tau(k)))


def _desc_pbc(R, N, lat, lat_inv):
    from sgdml_b200 import _lib

    B, D = R.shape[0], N * (N - 1) // 2
    x = np.full((B, D), np.nan)
    g = np.full((B, D, 3), np.nan)
    _lib.check(_lib.lib().sgdml_b200_desc_from_R_pbc(_lib.ptr(R), B, N, _lib.ptr(lat), _lib.ptr(lat_inv), _lib.ptr(x),
                                                     _lib.ptr(g), _lib.current_stream()), 'desc_from_R_pbc')
    return x, g


@pytest.mark.parametrize('N', [21, 60])
def test_desc_from_R_pbc_componentwise(eng, N):
    """(c) 1 000 geometries against the oracle's descriptors within predict_checks.desc_pbc_bound."""
    lat = np.ascontiguousarray(pc.skewed_cell(N))
    lat_inv = _lat_inv(lat)
    from sgdml_b200 import synth

    R = synth.geometries(N, 1100, 300 + N).reshape(1100, -1)
    keep = pc.pbc_margin(R, lat, lat_inv) >= MARGIN
    assert np.sum(~keep[:1000]) <= 50
    R = np.ascontiguousarray(R[keep][:1000])
    x, g = _desc_pbc(R, N, lat, lat_inv)
    x_ref, g_ref = odesc.from_R(R, (lat, lat_inv))
    bx, bg = pc.desc_pbc_bound(R, lat, lat_inv)
    ex = np.abs(x - x_ref) / bx
    eg = np.abs(g - g_ref) / bg[..., None]
    print('\n[desc bound] N=%d: max|err|/bound x %.2e g %.2e' % (N, np.max(ex), np.max(eg)))
    assert np.all(ex <= 1) and np.all(eg <= 1)


# (e) exact ties in a cubic cell of edge 8: pairs (1, 0), (3, 0) differ by +-4 along x, (2, 0), (5, 4) by +12 / -12,
# so lat_inv @ d is exactly +-0.5 or +-1.5 (dyadic coordinates, lat_inv = I / 8); rint and np.around both round half
# to even (0.5 -> 0, 1.5 -> 2), round-half-away would move the +-0.5 pairs to the other image
TIE_R0 = np.array([
    [0.0, 0.0, 0.0],
    [4.0, 0.5, 0.25],
    [12.0, 2.0, -0.5],
    [-4.0, -1.5, 1.0],
    [2.25, 3.0, 2.0],
    [-9.75, 3.0, 2.0],
])
TIE_PAIRS = {(1, 0): 0.5, (3, 0): -0.5, (2, 0): 1.5, (5, 4): -1.5}


def _tie_queries():
    """Three queries that keep every tie exact: R0, R0 translated by a dyadic vector, and R0 with atoms 4 and 5 moved
    together."""
    moved = np.zeros((6, 3))
    moved[4:] = [0.25, -0.25, 0.125]
    R = np.stack([TIE_R0, TIE_R0 + [0.5, -0.25, 0.125], TIE_R0 + moved])
    return np.ascontiguousarray(R.reshape(3, -1))


def test_exact_rounding_ties(eng, monkeypatch):
    N = 6
    lat = 8.0 * np.eye(3)
    lat_inv = np.eye(3) / 8.0
    R = _tie_queries()
    _, c = pc._pair_frac(R, lat_inv)
    a, b = np.tril_indices(N, -1)
    for d, (i, j) in enumerate(zip(a, b)):
        if (i, j) in TIE_PAIRS:
            assert np.all(c[:, d, 0] == TIE_PAIRS[(i, j)]) and np.all(np.abs(c[:, d, 1:] - np.floor(c[:, d, 1:]) - 0.5) >= 0.01)
        else:
            assert np.all(np.abs(c[:, d] - np.floor(c[:, d]) - 0.5) >= 0.01), (i, j)
    x_ref, g_ref = odesc.from_R(R, (lat, lat_inv))
    assert np.max(x_ref) <= 1.0
    # the descriptor kernel picks the oracle's image for every pair: each Jacobian row has the oracle's signs
    x, g = _desc_pbc(R, N, lat, lat_inv)
    assert np.array_equal(np.sign(g), np.sign(g_ref))
    bx, bg = pc.desc_pbc_bound(R, lat, lat_inv)
    assert np.all(np.abs(x - x_ref) <= bx) and np.all(np.abs(g - g_ref) <= bg[..., None])
    # predictions through the chunked path and both graph forms
    from sgdml_b200 import synth

    M = 20
    Rt = (TIE_R0[None] + 0.05 * np.random.default_rng(5).standard_normal((M, N, 3))).reshape(M, -1)
    xt, gt = odesc.from_R(Rt, (lat, lat_inv))
    perms = synth.rotor_swap_group(N, 1, 1)
    alphas = np.random.default_rng(6).standard_normal(M * 3 * N)
    model = {
        'type': 'm', 'z': np.ones(N, dtype=np.int64), 'R_desc': np.ascontiguousarray(xt.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(gt, alphas.reshape(M, -1)), 'alphas_F': alphas, 'c': 0.37, 'std': 1.7,
        'sig': SIG, 'lam': 1e-10, 'perms': perms, 'tril_perms_lin': odesc.tril_perms_lin(perms), 'use_E': True,
        'lattice': lat,
    }
    op = opredict.Predictor(model)
    with _env(monkeypatch, SGDML_B200_GRAPH='0'):
        E0, F0 = eng.GDMLPredict(model).predict(R)
    _check('ties chunked', model, op, R, range(3), E0, F0)
    for zc in ('1', '0'):
        with _env(monkeypatch, SGDML_B200_GRAPH='1', SGDML_B200_GRAPH_ZEROCOPY=zc):
            pg = eng.GDMLPredict(model)
            pg.predict(R[::-1].copy())  # captures
            E, F = pg.predict(R)  # replays
        assert np.array_equal(E, E0) and np.array_equal(F, F0), 'graph (zero copy %s) differs at the ties' % zc


# --------------------------------------------------------------------------- 4. graph invalidation on one handle
def _set_alphas_E_raw(p, ptr):
    from sgdml_b200 import _lib

    return _lib.lib().sgdml_b200_model_set_alphas_E(p._handle, ptr, _lib.current_stream())


def _set_lattice_raw(p, lat_ptr, inv_ptr):
    from sgdml_b200 import _lib

    return _lib.lib().sgdml_b200_model_set_lattice(p._handle, lat_ptr, inv_ptr)


def test_graph_invalidation_and_rejected_calls(eng, monkeypatch):
    """A class 3 handle (D = 153, split-k row-half exchange) created without alphas_E, with a graph captured at B = 3,
    then: alphas_E set, alphas_E switched off, alphas_E from a CUDA tensor through the C ABI, a new cell, no cell, and
    two rejected set_lattice calls on a periodic handle.  Each step toggles what the graph captured before it carries
    as a kernel argument (use_ae) or stages per call (the cell), so a graph that is not captured again, or that reads a
    stale cell, gives the old state's results.
    After each step the graph, the chunked path and K.v match the oracle of the handle's new state."""
    from sgdml_b200 import _lib

    torch = _torch()
    N, M, _ = SHAPES['c3']
    model, x, g = _make(N, M, seed=31, ecstr=True)
    aF = model['alphas_F']
    lat = np.ascontiguousarray(pc.skewed_cell(N))
    lat_inv = _lat_inv(lat)
    seed = [500]

    def fresh_R(B):
        seed[0] += 1
        return _queries(N, B, seed[0], lat)

    p = eng.GDMLPredict(dict((k, v) for k, v in model.items() if k != 'alphas_E'))
    p.set_R_desc(x)
    p.set_R_d_desc(g)
    p.set_alphas(aF)  # the handle's JA from here on comes from the device's J^T alpha, as in every later step
    p.predict(fresh_R(3))  # graph captured without energy constraints

    def routes(state, tag):
        """Graph and chunked routes (same inputs, bit-identical) and K.v against the oracle of `state`."""
        R3 = fresh_R(3)
        E, F = p.predict(R3)
        with _env(monkeypatch, SGDML_B200_GRAPH='0'):
            E0, F0 = p.predict(R3)
        assert np.array_equal(E, E0) and np.array_equal(F, F0), tag
        m = dict(model)
        m.pop('alphas_E')
        m.pop('lattice', None)
        if state.get('ae') is not None:
            m['alphas_E'] = state['ae']
        if state.get('lat') is not None:
            m['lattice'] = state['lat']
        _check('invalidation: %s' % tag, m, opredict.Predictor(m), R3, range(3), E, F)
        _check_kv(p, m, x, g, aF, state.get('ae'), [(0, M), (5, M - 7)], 'invalidation: %s' % tag)
        return E, F

    def like_fresh_handle(ae, R3, E, F):
        q = eng.GDMLPredict(dict((k, v) for k, v in model.items() if k != 'alphas_E'))
        q.set_R_desc(x)
        q.set_R_d_desc(g)
        q.set_alphas(aF, alphas_E=ae)
        E2, F2 = q.predict(R3)
        assert np.array_equal(E, E2) and np.array_equal(F, F2)

    # alphas_E set through set_alphas: the graph captured without them must not be replayed
    ae2 = 0.5 * np.random.default_rng(32).standard_normal(M)
    p.set_alphas(aF, alphas_E=ae2)
    routes({'ae': ae2}, 'set_alphas(alphas_F, alphas_E2)')
    # alphas_E off: bit-identical to a handle created without it
    assert _set_alphas_E_raw(p, None) == 0
    routes({}, 'set_alphas_E(NULL)')
    R3 = fresh_R(3)
    E, F = p.predict(R3)
    like_fresh_handle(None, R3, E, F)
    # alphas_E from device memory: the copy is ordered on the caller's stream, not synchronised
    ae3 = 0.5 * np.random.default_rng(33).standard_normal(M)
    t = torch.from_numpy(ae3).cuda()
    assert _set_alphas_E_raw(p, t.data_ptr()) == 0
    routes({'ae': ae3}, 'set_alphas_E(CUDA tensor)')
    # a new cell, then none: bit-identical to a free-molecule handle
    assert _set_lattice_raw(p, _lib.ptr(lat), _lib.ptr(lat_inv)) == 0
    routes({'ae': ae3, 'lat': lat}, 'set_lattice(cell)')
    assert _set_lattice_raw(p, None, None) == 0
    routes({'ae': ae3}, 'set_lattice(NULL)')
    R3 = fresh_R(3)
    E, F = p.predict(R3)
    like_fresh_handle(ae3, R3, E, F)
    # rejected calls on a periodic handle leave the cell as it was
    assert _set_lattice_raw(p, _lib.ptr(lat), _lib.ptr(lat_inv)) == 0
    R3 = fresh_R(3)
    E_before, F_before = p.predict(R3)
    assert _set_lattice_raw(p, _lib.ptr(lat), None) == ERR_ARG
    E, F = p.predict(R3)
    assert np.array_equal(E, E_before) and np.array_equal(F, F_before), 'a rejected set_lattice (one NULL) changed the model'
    lat_d, inv_d = torch.from_numpy(lat).cuda(), torch.from_numpy(lat_inv).cuda()
    assert _set_lattice_raw(p, lat_d.data_ptr(), inv_d.data_ptr()) == ERR_ARG
    E, F = p.predict(R3)
    assert np.array_equal(E, E_before) and np.array_equal(F, F_before), 'a rejected set_lattice (device) changed the model'
    routes({'ae': ae3, 'lat': lat}, 'after rejected set_lattice')


# --------------------------------------------------------------------------- 5. assembly and training
@pytest.mark.parametrize('N', [9, 21, 34, 60])
def test_assemble_ecstr_after_assemble(eng, N):
    """sgdml_b200_assemble then sgdml_b200_assemble_ecstr (the order the analytic solver's assembly uses) at scale -1
    into a padded row stride: against the oracle's energy-constrained matrix; the mirrored energy rows and columns
    bit-identical, the padding columns untouched."""
    from sgdml_b200 import _lib, synth

    torch = _torch()
    M, sig = 6, 30
    perms = synth.rotor_swap_group(N, 1, 1)
    lin = np.ascontiguousarray(odesc.tril_perms_lin(perms), dtype=np.int64)
    x, g = odesc.from_R(synth.geometries(N, M, 40 + N).reshape(M, -1))
    x, g = np.ascontiguousarray(x), np.ascontiguousarray(g)
    n = 3 * N * M
    n_tot, ldk = n + M, n + M + 3
    K = torch.full((n_tot, ldk), float('nan'), dtype=torch.float64, device='cuda')
    L = _lib.lib()
    S = perms.shape[0]
    st = _lib.current_stream()
    _lib.check(L.sgdml_b200_assemble(_lib.ptr(x), _lib.ptr(g), _lib.ptr(lin), N, M, S, float(sig), None, n, -1.0,
                                     K.data_ptr(), ldk, st), 'assemble')
    _lib.check(L.sgdml_b200_assemble_ecstr(_lib.ptr(x), _lib.ptr(g), _lib.ptr(lin), N, M, S, float(sig), -1.0,
                                           K.data_ptr(), ldk, st), 'assemble_ecstr')
    Kh = K.cpu().numpy()
    K_ref = -oassemble.assemble_E_cstr(x, g, lin, sig)
    assert rel_err(Kh[:, :n_tot], K_ref) < 1e-12
    assert rel_err(Kh[n:, n:n_tot], K_ref[n:, n:]) < 1e-12
    assert np.array_equal(Kh[n:, :n], Kh[:n, n:n_tot].T)
    assert np.all(np.isnan(Kh[:, n_tot:]))


def test_train_periodic_energy_constrained_vs_oracle(eng):
    """GDMLTrain.train with a lattice and use_E_cstr (analytic solver) against oracle.train at N = 15, M = 40."""
    from sgdml_b200 import synth

    N, M = 15, 40
    lat = pc.skewed_cell(N)
    task = synth.make_task(N, M, synth.rotor_swap_group(N, 1, 1), SIG)
    task['lattice'] = lat
    task['use_E_cstr'] = True
    model = eng.GDMLTrain().train(task)
    ref = otrain.train(task)
    assert 'alphas_E' in model and 'alphas_E' in ref and 'lattice' in model
    assert abs(float(model['c']) - float(ref['c'])) <= 1e-6 * abs(float(ref['c']))
    Rq = _queries(N, 20, 77, lat)
    E, F = eng.GDMLPredict(model).predict(Rq)
    E_ref, F_ref = opredict.Predictor(ref).predict(Rq)
    assert rel_err(F, F_ref) < 1e-6 and rel_err(E, E_ref) < 1e-6
