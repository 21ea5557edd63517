"""sgdml_b200_predict_virial / GDMLPredict.predict_virial on every finishing route against the oracle virial
(tests/virial_checks.py) with the componentwise bound check_W, and E / F against `predict` bit for bit.

Routes: k_predict_finish<true> with QPB > 1 (D <= 40) and QPB = 1, k_predict_finish_small<true> (graph-sized batches
whose sweep over the training points is split), the GEMM-composed path (D > 256), the long-descriptor pair
k_fdesc_gather<true> / k_fdesc_project<true> (N >= 227); batches through the zero-copy graph, the copy-node graph, plain
launches, several chunks and the pipelined host path; NumPy, pinned and CUDA-tensor I/O.  Cells given per call travel
with the geometries through the graph: a new cell replays the graph, which the launch counter of the main kernel shows
(a replay counts none).  Output buffers are NaN-filled first."""

import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import predict_checks as pc  # noqa: E402
import virial_checks as vc  # noqa: E402
from conftest import load_golden  # noqa: E402
from oracle import desc as odesc  # noqa: E402
from oracle import predict as opredict  # noqa: E402
from test_predict_bulk import _chunk_cap, _main_launches  # noqa: E402

ERR_ARG = -1000
# name: (N, M); D = 36 (QPB 3), 105 (QPB 1), 253, 276 (GEMM-composed)
SHAPES = {'d36': (9, 70), 'd105': (15, 41), 'd253': (23, 29), 'd276': (24, 19)}


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


@contextlib.contextmanager
def _env(monkeypatch, **kv):
    with monkeypatch.context() as mp:
        for k, v in kv.items():
            mp.setenv(k, v)
        yield


def _np(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def _check(tag, model, op, R, E, F, W):
    """E, F (check_predict) and W (check_W) against the oracle `op` (in the cell of the call)."""
    E, F, W = _np(E), _np(F), _np(W)
    E_ref, F_ref, W_ref, _ = vc.oracle_virial(op, R)
    D = model['R_desc'].shape[0]
    k = pc.n_terms(model['R_desc'].shape[1], op.n_perms, D)
    m = dict(model)
    if op.lat_and_inv is not None:
        m['lattice'] = op.lat_and_inv[0]
    else:
        m.pop('lattice', None)
    pc.check_predict(E, F, E_ref, F_ref, pc.predict_abs_scale(m, R, oracle=op), k, what=tag)
    r = vc.check_W(W, W_ref, vc.virial_abs_scale(m, R, op), k, what=tag)
    print('\n[virial bound] %s: %d rows, max|err|/scale %.2e, tau %.2e' % (tag, R.shape[0], r, pc.tau(k)))
    assert r <= pc.tau(k) / 10, 'less than 10x margin below tau'


def _same_as_predict(p, R, E, F, tag):
    E0, F0 = p.predict(R)
    assert np.array_equal(_np(E), E0) and np.array_equal(_np(F), F0), '%s: E / F differ from predict' % tag


def _nan(B, dim_i):
    return np.full(B, np.nan), np.full((B, dim_i), np.nan), np.full((B, 3, 3), np.nan)


def _routes(eng, monkeypatch, model, op, lat, tag, seed):
    """Every batch route of one model (cell `lat` per call; None: the model's own)."""
    import torch

    N = int(np.asarray(model['z']).shape[0])
    dim_i = 3 * N
    mlat = model.get('lattice')
    cell = lat if lat is not None else mlat
    Rq = lambda B, s: vc.queries(N, B, seed + s, cell)  # noqa: E731
    p = eng.GDMLPredict(model)
    # host B = 37 (plain launches), out= NaN-filled
    R = Rq(37, 0)
    out = _nan(37, dim_i)
    E, F, W = p.predict_virial(R, lattice=lat, out=out)
    assert E is out[0] and W is out[2]
    _check('%s host B=37' % tag, model, op, R, E, F, W)
    if lat is None:
        _same_as_predict(p, R, E, F, tag)
    # CUDA tensors B = 1 and 37, pinned host tensors B = 20
    for B, s in ((1, 1), (37, 2)):
        R = Rq(B, s)
        E, F, W = p.predict_virial(torch.from_numpy(R).cuda(), lattice=lat)
        torch.cuda.synchronize()
        assert W.is_cuda and W.shape == (B, 3, 3)
        _check('%s device B=%d' % (tag, B), model, op, R, E, F, W)
    R = Rq(20, 3)
    E, F, W = p.predict_virial(torch.from_numpy(R).pin_memory(), lattice=lat)
    assert W.is_pinned() and F.is_pinned()
    _check('%s pinned B=20' % tag, model, op, R, E, F, W)
    # several chunks of at most 5 queries
    with _chunk_cap(5):
        pc5 = eng.GDMLPredict(model)
        R = Rq(23, 4)
        E, F, W = pc5.predict_virial(R, lattice=lat)
    _check('%s host B=23 cap 5' % tag, model, op, R, E, F, W)
    # B = 1, 3, 16 through both graph forms and through plain launches: W bit-identical between them
    for B in (1, 3, 16):
        R = Rq(B, 10 + B)
        with _env(monkeypatch, SGDML_B200_GRAPH='0'):
            E0, F0, W0 = eng.GDMLPredict(model).predict_virial(R, lattice=lat)
        _check('%s host B=%d plain' % (tag, B), model, op, R, E0, F0, W0)
        for zc in ('1', '0'):
            with _env(monkeypatch, SGDML_B200_GRAPH='1', SGDML_B200_GRAPH_ZEROCOPY=zc):
                pg = eng.GDMLPredict(model)
                pg.predict_virial(Rq(B, 20 + B), lattice=lat)  # captures
                n0 = _main_launches()
                E, F, W = pg.predict_virial(R, lattice=lat, out=_nan(B, dim_i))  # replays
                assert _main_launches() == n0, 'graph not replayed'
                if lat is None:
                    _same_as_predict(pg, R, E, F, tag)
            assert np.array_equal(E, E0) and np.array_equal(F, F0) and np.array_equal(W, W0), \
                '%s B=%d: graph (zero copy %s) differs from plain launches' % (tag, B, zc)
    return p


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_virial_every_route_free(eng, monkeypatch, name):
    N, M = SHAPES[name]
    model = vc.make_model(N, M, seed=N)
    _routes(eng, monkeypatch, model, opredict.Predictor(model), None, 'free %s' % name, 100 + N)
    # free molecule: W equals sum_i r_i F_i^T of the same call
    p = eng.GDMLPredict(model)
    R = vc.queries(N, 9, 7)
    E, F, W = p.predict_virial(R)
    Wc = vc.classical_virial(R, F)
    assert np.max(np.abs(W - Wc)) <= 1e-10 * np.max(np.abs(W))


def test_virial_energy_constrained(eng, monkeypatch):
    N, M = SHAPES['d105']
    model = vc.make_model(N, M, seed=51, ecstr=True)
    _routes(eng, monkeypatch, model, opredict.Predictor(model), None, 'ecstr d105', 300)


@pytest.mark.parametrize('name', ['d36', 'd253', 'd276'])
def test_virial_periodic_skewed_cell(eng, monkeypatch, name):
    """A periodic model in a skewed cell that really wraps: its own cell, then a different cell per call."""
    N, M = SHAPES[name]
    lat = pc.skewed_cell(N)
    model = vc.make_model(N, M, seed=N + 1, lattice=lat)
    op = opredict.Predictor(model)
    R = vc.queries(N, 37, 400, lat)
    _, c = pc._pair_frac(R, np.linalg.inv(lat))
    assert np.mean(np.any(np.around(c) != 0, axis=-1)) >= 0.2
    p = _routes(eng, monkeypatch, model, op, None, 'pbc %s' % name, 400)
    # the model's own cell given per call: bit-identical to NULL
    E0, F0, W0 = p.predict_virial(R)
    E1, F1, W1 = p.predict_virial(R, lattice=lat)
    assert np.array_equal(E0, E1) and np.array_equal(F0, F1) and np.array_equal(W0, W1)
    # a different cell per call (the model keeps its own)
    lat2 = np.diag([1.07, 0.96, 1.03]) @ lat
    _routes(eng, monkeypatch, model, vc.with_cell(op, lat2), lat2, 'pbc %s cell2' % name, 500)
    E2, F2 = p.predict(R)
    assert np.array_equal(E2, E0) and np.array_equal(F2, F0), 'a per-call cell changed the model'


def test_virial_periodic_golden_pbc_n6_m8(eng, monkeypatch):
    """The reference-generated periodic fixture's model, its queries and its cell."""
    from conftest import golden_model

    g = load_golden('pbc_n6_m8')
    model = golden_model(g)
    model['lattice'] = g['lattice']
    op = opredict.Predictor(model)
    R = np.ascontiguousarray(g['R_query'])
    assert np.min(pc.pbc_margin(R, g['lattice'], np.linalg.inv(g['lattice']))) >= 1e-6
    p = eng.GDMLPredict(model)
    for B in (R.shape[0], 1, 3):
        E, F, W = p.predict_virial(R[:B])
        _check('pbc_n6_m8 B=%d' % B, model, op, R[:B], E, F, W)
        _same_as_predict(p, R[:B], E, F, 'pbc_n6_m8')
    _routes(eng, monkeypatch, model, op, None, 'pbc_n6_m8', 600)


def test_virial_long_descriptors_n240(eng):
    """N = 240, M = 2 (D = 28 680): k_fdesc_gather<true> / k_fdesc_project<true>, graph and plain batches and CUDA tensors."""
    import torch

    g = load_golden('big_n240_m2_s3')
    N = int(g['n_atoms'])
    S = g['perms'].shape[0]
    lin = odesc.tril_perms_lin(g['perms'])
    M = g['R_train'].shape[0]
    x, gd = odesc.from_R(g['R_train'].reshape(M, -1))
    model = {
        'type': 'm', 'z': g['z'], 'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(gd, g['alphas_F'].reshape(M, -1)), 'alphas_F': g['alphas_F'],
        'c': float(g['c']), 'std': float(g['std']), 'sig': int(g['sig']), 'lam': float(g['lam']), 'perms': g['perms'],
        'tril_perms_lin': lin, 'use_E': True,
    }
    assert S == 3
    op = opredict.Predictor(model)
    p = eng.GDMLPredict(model)
    R = np.ascontiguousarray(g['R_query'])
    fin0 = _lib_finish_launches()
    E, F, W = p.predict_virial(R)
    assert _lib_finish_launches() > fin0, 'the long-descriptor finishing pair did not run'
    _check('n240 B=%d' % R.shape[0], model, op, R, E, F, W)
    _same_as_predict(p, R, E, F, 'n240')
    Et, Ft, Wt = p.predict_virial(torch.from_numpy(R).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(_np(Wt), W)
    E1, F1, W1 = p.predict_virial(R[:1])
    assert np.array_equal(W1, W[:1])


def _lib_finish_launches():
    from sgdml_b200 import _lib

    return _lib.profile_snapshot()['predict_finish'][2]


def test_virial_pipelined_host_batch(eng):
    """B = 4100 host queries: the pipelined path on two streams (four chunks of 1025), E / F bit-identical to `predict`
    on the same path; chunk edges and sampled rows against the oracle, as are those of the same batch as CUDA tensors
    (one chunk, whose main kernel splits the sweep over M differently: the two agree within the bound, not bit for
    bit)."""
    import torch

    N, M = SHAPES['d36']
    model = vc.make_model(N, M, seed=71)
    op = opredict.Predictor(model)
    B = 4100
    R = vc.queries(N, B, 72)
    p = eng.GDMLPredict(model)
    E, F, W = p.predict_virial(R)
    _same_as_predict(p, R, E, F, 'pipelined')
    rows = np.unique(np.concatenate([[0, 1024, 1025, 2049, 3075, B - 1],
                                     np.random.default_rng(3).choice(B, 40, replace=False)]))
    _check('pipelined B=4100 (%d rows)' % len(rows), model, op, R[rows], E[rows], F[rows], W[rows])
    Ed, Fd, Wd = p.predict_virial(torch.from_numpy(R).cuda())
    torch.cuda.synchronize()
    _check('device B=4100 (%d rows)' % len(rows), model, op, R[rows], _np(Ed)[rows], _np(Fd)[rows], _np(Wd)[rows])


def test_cell_changes_replay_without_capture(eng):
    """Consecutive B = 1 calls, each with a new cell: correct W every time, and after the first capture every call
    replays the graph (no main-kernel launch is counted for a replay)."""
    N, M = SHAPES['d36']
    lat = pc.skewed_cell(N)
    model = vc.make_model(N, M, seed=81, lattice=lat)
    op = opredict.Predictor(model)
    p = eng.GDMLPredict(model)
    p.predict_virial(vc.queries(N, 1, 80, lat), lattice=lat)  # captures
    n0 = _main_launches()
    for i in range(6):
        L = (1.0 + 0.01 * i) * lat + 0.02 * i * np.eye(3)
        R = vc.queries(N, 1, 90 + i, L)
        E, F, W = p.predict_virial(R, lattice=L)
        _check('cell change %d' % i, model, vc.with_cell(op, L), R, E, F, W)
    assert _main_launches() == n0, 'a new cell recaptured the graph'


def test_set_lattice_replays_the_graph(eng):
    """No cell is baked into a graph: B = 3 graphs of `predict_virial` and `predict` captured on a periodic handle
    replay after set_lattice with a new cell, and after set_lattice(NULL, NULL), and match the oracle in the handle's
    cell of the moment (E and F of `predict` bit for bit)."""
    from sgdml_b200 import _lib

    N, M = SHAPES['d36']
    lat = pc.skewed_cell(N)
    model = vc.make_model(N, M, seed=85, lattice=lat)
    op = opredict.Predictor(model)
    p = eng.GDMLPredict(model)
    R = vc.queries(N, 3, 86, lat)
    p.predict_virial(R)  # captures
    p.predict(R)  # captures
    n0 = _main_launches()
    lat2 = np.ascontiguousarray(np.diag([1.07, 0.96, 1.03]) @ lat)
    for cell, seed in ((lat2, 87), (None, 88)):
        if cell is None:
            rc = _lib.lib().sgdml_b200_model_set_lattice(p._handle, None, None)
        else:
            rc = _lib.lib().sgdml_b200_model_set_lattice(p._handle, _lib.ptr(cell),
                                                         _lib.ptr(np.ascontiguousarray(np.linalg.inv(cell))))
        assert rc == 0
        R = vc.queries(N, 3, seed, cell)
        E, F, W = p.predict_virial(R)
        _check('set_lattice(%s)' % ('NULL' if cell is None else 'cell'), model, vc.with_cell(op, cell), R, E, F, W)
        _same_as_predict(p, R, E, F, 'set_lattice')
        assert _main_launches() == n0, 'set_lattice recaptured the graph'


def test_int8_slice_route_classical_identity(eng):
    """The int8-slice contractions of D > 256 (5 slices): W equals sum_i r_i F_i^T of the same call."""
    N, M = SHAPES['d276']
    model = vc.make_model(N, M, seed=91)
    p = eng.GDMLPredict(model)
    p.set_contraction_slices(5)
    R = vc.queries(N, 21, 92)
    E, F, W = p.predict_virial(R)
    Wc = vc.classical_virial(R, F)
    rel = np.max(np.abs(W - Wc)) / np.max(np.abs(W))
    print('\n[virial] int8 slices: max|W - sum r F^T|/max|W| %.1e' % rel)
    assert rel <= 1e-10


def test_rejected_calls_leave_the_model(eng):
    """Singular, non-finite, half-NULL and device-pointer cells are rejected; the model's cell and its captured graph
    stay as they were (the next call replays it and gives the same results)."""
    import torch

    from sgdml_b200 import _lib

    N, M = SHAPES['d36']
    lat = np.ascontiguousarray(pc.skewed_cell(N))
    model = vc.make_model(N, M, seed=95, lattice=lat)
    p = eng.GDMLPredict(model)
    R = vc.queries(N, 1, 96, lat)
    E0, F0, W0 = p.predict_virial(R)
    n0 = _main_launches()
    E = np.empty(1)
    F = np.empty((1, 3 * N))
    W = np.empty((1, 3, 3))
    lat_inv = np.ascontiguousarray(np.linalg.inv(lat))
    sing = np.ascontiguousarray(np.outer([1.0, 2.0, 3.0], [1.0, 0.5, 0.25]))
    nanc = lat.copy()
    nanc[1, 1] = np.nan
    lat_d = torch.from_numpy(lat).cuda()
    inv_d = torch.from_numpy(lat_inv).cuda()
    L = _lib.lib()
    st = _lib.current_stream()
    for a, b in ((_lib.ptr(sing), _lib.ptr(lat_inv)), (_lib.ptr(nanc), _lib.ptr(lat_inv)), (_lib.ptr(lat), None),
                 (lat_d.data_ptr(), inv_d.data_ptr())):
        rc = L.sgdml_b200_predict_virial(p._handle, _lib.ptr(R), 1, a, b, _lib.ptr(E), _lib.ptr(F), _lib.ptr(W), st)
        assert rc == ERR_ARG
    assert L.sgdml_b200_predict_virial(p._handle, _lib.ptr(R), 1, None, None, _lib.ptr(E), _lib.ptr(F), None, st) == ERR_ARG
    E1, F1, W1 = p.predict_virial(R)
    assert _main_launches() == n0, 'a rejected call dropped the captured graph'
    assert np.array_equal(E1, E0) and np.array_equal(F1, F0) and np.array_equal(W1, W0)
    E2, F2 = p.predict(R)
    assert np.array_equal(E2, E0) and np.array_equal(F2, F0)


def test_ase_core_stress(eng):
    """SGDMLCalculatorCore: stress = -W E_to_eV / V (Voigt) of the model's own cell and of the atoms' cell; a central
    difference of the core's energy under strain (cell given as ASE rows in Angstrom) matches it; free-molecule models
    refuse stress."""
    from sgdml_b200.intf.ase_calc import SGDMLCalculatorCore

    N, M = SHAPES['d36']
    lat = pc.skewed_cell(N)
    model = vc.make_model(N, M, seed=97, lattice=lat)
    E_to_eV, F_to_eV_Ang = 0.0433641, 0.0433641 / 1.1  # model length unit = 1.1 Angstrom
    Ang_to_R = F_to_eV_Ang / E_to_eV
    core = SGDMLCalculatorCore()
    core._setup(model, E_to_eV, F_to_eV_Ang, use_atoms_cell=True)
    assert 'stress' in core.implemented_properties
    R = vc.queries(N, 1, 98, lat)
    pos = R.reshape(N, 3) / Ang_to_R  # Angstrom
    cell = lat.T / Ang_to_R  # ASE rows, Angstrom
    res = core.compute(pos, cell=cell, stress=True)
    # the same call in model units: positions * Ang_to_R, the cell transposed to columns * Ang_to_R
    _, _, W = core.gdml_predict.predict_virial((pos * Ang_to_R).ravel(), lattice=cell.T * Ang_to_R)
    s = -W[0] * E_to_eV / abs(np.linalg.det(cell))
    voigt = np.array([s[0, 0], s[1, 1], s[2, 2], s[1, 2], s[0, 2], s[0, 1]])
    assert np.allclose(res['stress'], voigt, rtol=1e-15, atol=0)
    res0 = core.compute(pos, stress=True)  # the model's own cell: the same numbers up to the unit round trip
    assert np.allclose(res0['stress'], res['stress'], rtol=1e-12, atol=0)
    # finite differences of the core's energy: sigma_ij = (1/V) dE/d(eps_ij)
    h = 1e-5
    fd = np.empty(6)
    for n, (i, j) in enumerate(vc.STRAINS):
        e = np.zeros((3, 3))
        e[i, j] += 0.5
        e[j, i] += 0.5

        def energy(t):
            A = np.eye(3) + t * e
            return core.compute(pos @ A.T, cell=cell @ A.T)['energy'][0]

        d1 = (energy(h) - energy(-h)) / (2 * h)
        d2 = (energy(h / 2) - energy(-h / 2)) / h
        fd[n] = (4 * d2 - d1) / 3 / abs(np.linalg.det(cell))
    rel = np.max(np.abs(fd - res['stress'])) / np.max(np.abs(res['stress']))
    print('\n[ase stress] finite-difference stress vs core: %.1e' % rel)
    assert rel < 1e-6
    # free molecules have no stress
    free = SGDMLCalculatorCore()
    free._setup(vc.make_model(N, M, seed=99), E_to_eV, F_to_eV_Ang)
    assert 'stress' not in free.implemented_properties
    with pytest.raises(ValueError, match='periodic'):
        free.compute(pos, stress=True)
