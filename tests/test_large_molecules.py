"""Molecules with hundreds of atoms: the predictor's finishing path for descriptors beyond its shared memory
(k_fdesc_gather / k_fdesc_project, N >= 227) and the energy-constraint assembly above 128 atoms, against the
reference's own outputs (tests/golden/big_n240_m2_s3.npz, big_n370_m2_s3.npz: synthetic molecules, M = 2, S = 3,
descriptor arrays and tril_perms_lin rows kept at a stride; tests/golden/make_golden_big.py) and the oracle."""

import numpy as np
import pytest

from conftest import load_golden, rel_err

from oracle import assemble as oassemble
from oracle import desc as odesc
from oracle import predict as opredict
from oracle import train as otrain

BIG = ['big_n240_m2_s3', 'big_n370_m2_s3']


def _load(name):
    """A fixture with the full tril_perms_lin: the oracle's, which must equal the reference's rows kept in the file."""
    g = load_golden(name)
    lin = odesc.tril_perms_lin(g['perms'])
    S = g['perms'].shape[0]
    assert np.array_equal(lin.reshape(-1, S)[g['desc_idx']], g['tril_perms_lin_sub'])
    g['tril_perms_lin'] = lin
    return g


def _oracle_desc(g):
    M = g['R_train'].shape[0]
    return odesc.from_R(g['R_train'].reshape(M, -1))


def _model(g, x, gd, alphas_E=None):
    """The fixture's random-coefficient model (reference layout) on the given training descriptors."""
    M = x.shape[0]
    m = {
        'type': 'm',
        'z': g['z'],
        'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(gd, g['alphas_F'].reshape(M, -1)),
        'alphas_F': g['alphas_F'],
        'c': float(g['c']),
        'std': float(g['std']),
        'sig': int(g['sig']),
        'lam': float(g['lam']),
        'perms': g['perms'],
        'tril_perms_lin': g['tril_perms_lin'],
        'use_E': True,
    }
    if alphas_E is not None:
        m['alphas_E'] = alphas_E
    return m


# --------------------------------------------------------------------------- oracle (CPU)
@pytest.mark.parametrize('name', BIG)
def test_oracle_descriptors_and_predictions(name):
    g = _load(name)
    idx = g['desc_idx']
    x, gd = _oracle_desc(g)
    assert rel_err(x[:, idx], g['R_desc_sub']) < 1e-13 and rel_err(gd[:, idx], g['R_d_desc_sub']) < 1e-13
    model = _model(g, x, gd)
    assert rel_err(model['R_d_desc_alpha'][:, idx], g['R_d_desc_alpha_sub']) < 1e-13
    E, F = opredict.Predictor(model).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 1e-10 and rel_err(E, g['E_query']) < 1e-10
    if 'alphas_E' in g:
        E, F = opredict.Predictor(_model(g, x, gd, g['alphas_E'])).predict(g['R_query'])
        assert rel_err(F, g['F_query_ecstr']) < 1e-10 and rel_err(E, g['E_query_ecstr']) < 1e-10


def test_oracle_kernel_columns_n240():
    g = _load('big_n240_m2_s3')
    x, gd = _oracle_desc(g)
    sig = int(g['sig'])
    K = oassemble.assemble(x, gd, g['tril_perms_lin'], sig, col_idxs=g['cols'])
    assert rel_err(K, g['K_cols']) < 1e-12
    Ke = oassemble.assemble_E_cstr(x, gd, g['tril_perms_lin'], sig)[:, g['ecols']]
    assert rel_err(Ke, g['K_ecols']) < 1e-12


# --------------------------------------------------------------------------- engine (GPU)
@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


def _eng_desc(eng, g):
    from sgdml_b200.desc import Desc

    M = g['R_train'].shape[0]
    return Desc(int(g['n_atoms'])).from_R(g['R_train'].reshape(M, -1))


def _finish_launches():
    from sgdml_b200 import _lib

    return _lib.profile_snapshot()['predict_finish'][2]


@pytest.mark.gpu
@pytest.mark.parametrize('name', BIG)
def test_descriptors_and_kernel_columns(eng, name):
    """Descriptors, tril_perms_lin, the K column subset (k_assemble_large) and the energy-constraint columns, both the
    column-subset form (k_assemble_ecstr_rows) and the full matrix (k_assemble_ecstr), against the reference."""
    from sgdml_b200.desc import Desc

    g = _load(name)
    N, idx, sig = int(g['n_atoms']), g['desc_idx'], int(g['sig'])
    assert np.array_equal(eng.desc.tril_perms_lin(g['perms']), g['tril_perms_lin'])  # reference rows checked by _load
    x, gd = _eng_desc(eng, g)
    assert rel_err(x[:, idx], g['R_desc_sub']) < 1e-14 and rel_err(gd[:, idx], g['R_d_desc_sub']) < 1e-14
    t = eng.GDMLTrain()
    K = t._assemble_kernel_mat(x, gd, g['tril_perms_lin'], sig, Desc(N), col_idxs=g['cols'])
    assert rel_err(K, g['K_cols']) < 1e-11
    Ke = t._assemble_kernel_mat(x, gd, g['tril_perms_lin'], sig, Desc(N), use_E_cstr=True, col_idxs=g['ecols'])
    assert rel_err(Ke, g['K_ecols']) < 1e-11
    K_full = t._assemble_kernel_mat(x, gd, g['tril_perms_lin'], sig, Desc(N), use_E_cstr=True)
    assert rel_err(K_full[:, g['ecols']], g['K_ecols']) < 1e-11
    n = K_full.shape[0] - x.shape[0]
    assert np.array_equal(K_full[n:, :n], K_full[:n, n:].T)


@pytest.mark.gpu
@pytest.mark.parametrize('name', BIG)
def test_predict_every_route(eng, monkeypatch, name):
    """Predictions through every caller of the finishing path against the reference: bulk (device tensors), B = 1 and
    B = 16 through the CUDA graph (bit-identical to SGDML_B200_GRAPH=0), predict(R=None), raw kmatvec_train and a
    multi-chunk batch; the finishing kernels run (their own profile family) and repeat bit for bit."""
    import torch

    from sgdml_b200 import _lib

    g = _load(name)
    x, gd = _eng_desc(eng, g)
    model = _model(g, x, gd)
    Rq = g['R_query']
    L = _lib.lib()
    p = eng.GDMLPredict(model)
    n0 = _finish_launches()
    E, F = p.predict(torch.from_numpy(Rq).cuda())
    assert _finish_launches() == n0 + 2
    E, F = E.cpu().numpy(), F.cpu().numpy()
    assert rel_err(F, g['F_query']) < 1e-9 and rel_err(E, g['E_query']) < 1e-9
    for _ in range(2):  # run to run: bit-identical
        E2, F2 = p.predict(torch.from_numpy(Rq).cuda())
        assert np.array_equal(E2.cpu().numpy(), E) and np.array_equal(F2.cpu().numpy(), F)

    # small host batches: the graph path against the plain launches of the same call
    R16 = np.concatenate([Rq, np.tile(Rq, (7, 1)) + 0.01 * np.random.default_rng(5).standard_normal((14, Rq.shape[1]))])
    for B in (1, 16):
        with monkeypatch.context() as mp:
            mp.setenv('SGDML_B200_GRAPH', '0')
            E0, F0 = eng.GDMLPredict(model).predict(R16[:B])
        pg = eng.GDMLPredict(model)
        pg.predict(R16[:B] + 0.02)  # captures
        Eg, Fg = pg.predict(R16[:B])  # replays
        assert np.array_equal(Eg, E0) and np.array_equal(Fg, F0), 'graph replay differs at B = %d' % B
    assert rel_err(F0[:2], g['F_query']) < 1e-9 and rel_err(E0[:2], g['E_query']) < 1e-9

    # sixteen chunks of one query each (device tensors: the chunked path)
    assert L.sgdml_b200_set_predict_chunk(1) == 0
    try:
        Ec, Fc = eng.GDMLPredict(model).predict(torch.from_numpy(R16).cuda())
    finally:
        L.sgdml_b200_set_predict_chunk(0)
    assert rel_err(Fc.cpu().numpy(), F0) < 1e-12 and rel_err(Ec.cpu().numpy(), E0) < 1e-12

    # training points: predict(R=None) against predict(R_train), raw K.v against the scaled sums
    M = x.shape[0]
    p.set_R_desc(x)
    p.set_R_d_desc(gd)
    Et, Ft = p.predict()
    Eq, Fq = p.predict(g['R_train'].reshape(M, -1))
    assert rel_err(Ft, Fq) < 1e-12 and rel_err(Et, Eq) < 1e-12
    Fr, Er = np.full_like(Ft, np.nan), np.full(M, np.nan)
    p.kmatvec_train(0, M, out=Fr, E_out=Er)
    std, c = float(g['std']), float(g['c'])
    assert rel_err(Fr * std, Ft) < 1e-14 and rel_err(Er * std + c, Et) < 1e-14


@pytest.mark.gpu
@pytest.mark.parametrize('name', BIG)
def test_kmatvec_is_assembled_matrix_times_v(eng, name):
    """K.v through the predictor (what every CG iteration runs) against the engine-assembled energy-constrained
    matrix times v: K v = [F; -E]."""
    from sgdml_b200.desc import Desc

    g = _load(name)
    x, gd = _eng_desc(eng, g)
    M, N = x.shape[0], int(g['n_atoms'])
    K = eng.GDMLTrain()._assemble_kernel_mat(x, gd, g['tril_perms_lin'], int(g['sig']), Desc(N), use_E_cstr=True)
    rng = np.random.default_rng(N)
    vF, vE = rng.standard_normal(M * 3 * N), rng.standard_normal(M)
    p = eng.GDMLPredict(dict(_model(g, x, gd), std=1.0, c=0.0))
    p.set_R_desc(x)
    p.set_R_d_desc(gd)
    p.set_alphas(vF, vE)
    F, E = np.full((M, 3 * N), np.nan), np.full(M, np.nan)
    p.kmatvec_train(0, M, out=F, E_out=E)
    Kv = K @ np.concatenate([vF, vE])
    assert rel_err(F.ravel(), Kv[: M * 3 * N]) < 1e-10
    assert rel_err(-E, Kv[M * 3 * N :]) < 1e-10


@pytest.mark.gpu
def test_energy_constrained_model_predictions(eng):
    g = _load('big_n240_m2_s3')
    x, gd = _eng_desc(eng, g)
    E, F = eng.GDMLPredict(_model(g, x, gd, g['alphas_E'])).predict(g['R_query'])
    assert rel_err(F, g['F_query_ecstr']) < 1e-9 and rel_err(E, g['E_query_ecstr']) < 1e-9


def _task(N, M):
    from sgdml_b200 import synth

    return synth.make_task(N, M, synth.rotor_swap_group(N, 1, 0), 50)


@pytest.mark.gpu
@pytest.mark.parametrize('ecstr', [False, True])
def test_analytic_training_n240_vs_oracle(eng, ecstr):
    """GDMLTrain.train (analytic solver: assembly, energy constraints, Cholesky, integration constant through
    predict(R=None)) at N = 240 against oracle.train (M = 2: the oracle's dense Jacobians take minutes at M = 3)."""
    N, M = 240, 2
    task = _task(N, M)
    task['use_E_cstr'] = ecstr
    model = eng.GDMLTrain().train(task)
    ref = otrain.train(task)
    assert ('alphas_E' in model) == ecstr
    assert abs(float(model['c']) - float(ref['c'])) <= 1e-6 * abs(float(ref['c']))
    from sgdml_b200 import synth

    Rq = synth.geometries(N, 4, 9).reshape(4, -1)
    E, F = eng.GDMLPredict(model).predict(Rq)
    E_ref, F_ref = opredict.Predictor(ref).predict(Rq)
    assert rel_err(F, F_ref) < 1e-6 and rel_err(E, E_ref) < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize('ecstr', [False, True])
def test_iterative_training_n370(eng, ecstr):
    """The Nystroem-preconditioned CG at N = 370 (forced by a small memory budget: one inducing point of four): it
    converges, and its model predicts what the analytic model of the same task predicts, within solver tolerance."""
    from sgdml_b200 import synth

    N, M = 370, 4
    task = _task(N, M)
    task['use_E_cstr'] = ecstr
    np.random.seed(2)
    model = eng.GDMLTrain(max_memory=0.1).train(task)
    assert model['solver_name'] == 'cg' and 0 < int(model['solver_iters']) < 3 * N * M * 10  # below maxiter: converged
    assert ('alphas_E' in model) == ecstr
    exact = eng.GDMLTrain().train(task)
    assert exact['solver_name'] == 'analytic'
    Rq = synth.geometries(N, 4, 9).reshape(4, -1)
    E, F = eng.GDMLPredict(model).predict(Rq)
    Ex, Fx = eng.GDMLPredict(exact).predict(Rq)
    assert rel_err(F, Fx) < 5e-3 and rel_err(E, Ex) < 5e-3


@pytest.mark.gpu
def test_ase_calculator_n370(eng):
    """The ASE calculator (one geometry per call: the graph path) on the 370-atom molecule."""
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV, SGDMLCalculatorCore

    g = _load('big_n370_m2_s3')
    x, gd = _eng_desc(eng, g)
    calc = SGDMLCalculatorCore()
    calc._setup(_model(g, x, gd), _KCAL_PER_MOL_IN_EV, _KCAL_PER_MOL_IN_EV)
    for q in range(2):
        res = calc.compute(g['R_query'][q].reshape(-1, 3))
        assert rel_err(res['forces'].ravel(), g['F_query'][q] * _KCAL_PER_MOL_IN_EV) < 1e-9
        assert rel_err(res['energy'], g['E_query'][q : q + 1] * _KCAL_PER_MOL_IN_EV) < 1e-9
