"""GPU parity tests proper: every hot-path entry point of the C ABI against the oracle and
against the reference's golden outputs.  Tolerances: integer work bit-exact; floating point
far inside the 1e-6 relative bound of BASELINE.json's north_star (stated per test)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from conftest import golden_model, golden_task, load_golden, rel_err  # noqa: E402

import oracle  # noqa: E402,F401
from oracle import assemble as oassemble  # noqa: E402
from oracle import desc as odesc  # noqa: E402
from oracle import predict as opredict  # noqa: E402
from oracle import solve as osolve  # noqa: E402
from oracle import train as otrain  # noqa: E402


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


def _oracle_model(N, M, perms, sig, seed=0, alpha_scale=1.0):
    """Random-coefficient model built with the ORACLE's descriptor code (no GPU involved)."""
    from sgdml_b200 import synth

    R = synth.geometries(N, M, seed).reshape(M, -1)
    rng = np.random.default_rng(seed + 99)
    alphas = alpha_scale * rng.standard_normal(M * 3 * N)
    x, g = odesc.from_R(R)
    return (
        {
            'type': 'm',
            'z': np.ones(N, dtype=np.int64),
            'R_desc': x.T.copy(),
            'R_d_desc_alpha': odesc.d_desc_dot_vec(g, alphas.reshape(M, -1)),
            'alphas_F': alphas,
            'c': 0.37,
            'std': 1.7,
            'sig': sig,
            'lam': 1e-10,
            'perms': np.asarray(perms, dtype=np.int64),
            'tril_perms_lin': odesc.tril_perms_lin(perms),
            'use_E': True,
        },
        x,
        g,
    )


# --------------------------------------------------------------------------- representation
def test_tril_perms_lin_bit_exact(eng, golden):
    from sgdml_b200.desc import Desc, tril_perms_lin

    out = tril_perms_lin(golden['perms'])
    assert out.dtype == np.int64
    assert np.array_equal(out, golden['tril_perms_lin'])
    D = golden['R_desc'].shape[1]
    for p_idx, p in enumerate(golden['perms']):
        assert np.array_equal(Desc.perm(p), golden['tril_perms_lin'].reshape(D, -1)[:, p_idx] - p_idx * D)


def test_descriptor_golden(eng, golden):
    from sgdml_b200.desc import Desc

    N = int(golden['n_atoms'])
    M = golden['R_train'].shape[0]
    d = Desc(N)
    x, g = d.from_R(golden['R_train'].reshape(M, -1))
    assert rel_err(x, golden['R_desc']) < 1e-14
    assert rel_err(g, golden['R_d_desc']) < 1e-14
    # single geometry returns (D,), (D, 3) like desc.py:329-330
    x1, g1 = d.from_R(golden['R_train'][0].reshape(-1))
    assert x1.shape == (d.dim,) and g1.shape == (d.dim, 3)
    rng = np.random.default_rng(1)
    v = rng.standard_normal((M, 3 * N))
    assert rel_err(d.d_desc_dot_vec(golden['R_d_desc'], v), odesc.d_desc_dot_vec(golden['R_d_desc'], v)) < 1e-13
    w = rng.standard_normal((M, d.dim))
    assert rel_err(d.vec_dot_d_desc(golden['R_d_desc'], w), odesc.vec_dot_d_desc(golden['R_d_desc'], w)) < 1e-13


# --------------------------------------------------------------------------- predictor
def test_predict_golden(eng, golden):
    """E, F within 1e-6 rel of the reference NumPy path (north_star); we demand 1e-10."""
    p = eng.GDMLPredict(golden_model(golden))
    E, F = p.predict(golden['R_query'])
    assert rel_err(F, golden['F_query']) < 1e-10
    assert rel_err(E, golden['E_query']) < 1e-10
    M = golden['R_train'].shape[0]
    E, F = p.predict(golden['R_train'].reshape(M, -1))  # self terms (delta = 0)
    assert rel_err(F, golden['F_train_pred']) < 1e-10
    assert rel_err(E, golden['E_train_pred']) < 1e-10
    (F2,) = p.predict(golden['R_query'][0], return_E=False)  # 1-D input gets a leading axis
    assert F2.shape == (1, golden['R_query'].shape[1])
    assert rel_err(F2[0], golden['F_query'][0]) < 1e-10


@pytest.mark.parametrize(
    'N,M,rot,swap,sig',
    [
        (3, 5, 1, 0, 5),  # D = 3, S = 3
        (4, 70, 0, 2, 10),  # D = 6, S = 4, M not a multiple of any tile
        (9, 200, 1, 1, 20),  # BASELINE config 1 shape
        (12, 33, 1, 2, 30),  # D = 66 -> DP 72
        (15, 40, 2, 0, 30),  # D = 105 -> DP 112
        (18, 21, 1, 1, 40),  # D = 153 -> DP 160
        (21, 50, 1, 1, 20),  # BASELINE config 2 descriptor, D = 210 -> DP 224
        (23, 19, 0, 1, 20),  # D = 253 -> DP 256
        (24, 30, 1, 1, 30),  # D = 276 > 256 -> GEMM-composed large-descriptor path
        (42, 25, 2, 0, 50),  # BASELINE config 3 descriptor (D = 861), S = 9
    ],
)
def test_predict_vs_oracle_shapes(eng, N, M, rot, swap, sig):
    from sgdml_b200 import synth

    perms = synth.rotor_swap_group(N, rot, swap)
    model, _, _ = _oracle_model(N, M, perms, sig, seed=N)
    B = 37
    Rq = synth.geometries(N, B, 1).reshape(B, -1)
    E_ref, F_ref = opredict.Predictor(model).predict(Rq)
    p = eng.GDMLPredict(model)
    E, F = p.predict(Rq)
    assert rel_err(F, F_ref) < 1e-10
    assert rel_err(E, E_ref) < 1e-10
    E1, F1 = p.predict(Rq[:1])  # one geometry: the sweep over the training points split across CTAs
    assert rel_err(F1, F_ref[:1]) < 1e-10
    assert rel_err(E1, E_ref[:1]) < 1e-10


def test_predict_torch_device_tensors(eng):
    import torch
    from sgdml_b200 import synth

    N, M = 9, 64
    perms = synth.rotor_swap_group(N, 1, 1)
    model, _, _ = _oracle_model(N, M, perms, 20)
    Rq = synth.geometries(N, 300, 1).reshape(300, -1)
    p = eng.GDMLPredict(model)
    E_h, F_h = p.predict(Rq)
    E_d, F_d = p.predict(torch.from_numpy(Rq).cuda())
    assert E_d.is_cuda and F_d.is_cuda
    assert np.array_equal(E_d.cpu().numpy(), E_h) and np.array_equal(F_d.cpu().numpy(), F_h)


def test_permutation_equivariance(eng):
    """F(R[:, p, :]) == F(R)[:, p, :] and E invariant for every perm of the model group (SURVEY 4.5)."""
    from sgdml_b200 import synth

    N, M = 9, 50
    perms = synth.rotor_swap_group(N, 1, 1)
    model, _, _ = _oracle_model(N, M, perms, 20)
    p = eng.GDMLPredict(model)
    R = synth.geometries(N, 8, 3)
    E0, F0 = p.predict(R.reshape(8, -1))
    for pm in perms:
        E1, F1 = p.predict(R[:, pm, :].reshape(8, -1))
        assert rel_err(E1, E0) < 1e-12
        assert rel_err(F1.reshape(8, N, 3), F0.reshape(8, N, 3)[:, pm, :]) < 1e-11


def test_force_is_minus_energy_gradient(eng):
    from sgdml_b200 import synth

    N, M = 6, 30
    perms = synth.rotor_swap_group(N, 1, 0)
    model, _, _ = _oracle_model(N, M, perms, 10)
    p = eng.GDMLPredict(model)
    R = synth.geometries(N, 1, 4).reshape(1, -1)
    _, F = p.predict(R)
    h = 1e-5
    Rp = np.repeat(R, 6 * N, axis=0)
    for k in range(3 * N):
        Rp[2 * k, k] += h
        Rp[2 * k + 1, k] -= h
    E, _ = p.predict(Rp)
    grad = (E[0::2] - E[1::2]) / (2 * h)
    assert rel_err(-grad, F[0]) < 1e-7


def test_kv_identity_and_set_alphas(eng, golden):
    """K @ v == predict_train(alphas = v) (iterative.py:183-204), via set_R_d_desc / set_alphas."""
    m = golden_model(golden)
    p = eng.GDMLPredict(m)
    p.set_R_desc(golden['R_desc'])
    p.set_R_d_desc(golden['R_d_desc'])
    p.set_alphas(golden['v'])
    Kv = p.kmatvec_train().ravel()
    assert rel_err(Kv, golden['Kv']) < 1e-10
    ja = p.get_R_d_desc_alpha()
    N = int(golden['n_atoms'])
    assert rel_err(ja, odesc.d_desc_dot_vec(golden['R_d_desc'], golden['v'].reshape(-1, 3 * N))) < 1e-13
    # a slice of training points
    M = golden['R_desc'].shape[0]
    part = p.kmatvec_train(1, M - 1).ravel()
    assert rel_err(part, golden['Kv'][3 * N : (M - 1) * 3 * N]) < 1e-10
    # back to the trained coefficients: predict() with R=None == reference prediction on training points
    p.set_alphas(golden['alphas_F'])
    E, F = p.predict()
    assert rel_err(F, golden['F_train_pred']) < 1e-10
    assert rel_err(E, golden['E_train_pred']) < 1e-10


def test_predict_empty_and_errors(eng, golden):
    p = eng.GDMLPredict(golden_model(golden))
    N = int(golden['n_atoms'])
    E, F = p.predict(np.empty((0, 3 * N)))
    assert E.shape == (0,) and F.shape == (0, 3 * N)
    with pytest.raises(ValueError):
        p.predict(np.zeros((2, 3 * N + 1)))
    with pytest.raises(RuntimeError):
        eng.GDMLPredict(golden_model(golden)).predict()  # no cached training descriptors
    bad = golden_model(golden)
    bad['type'] = 'd'
    with pytest.raises(ValueError):
        eng.GDMLPredict(bad)


# --------------------------------------------------------------------------- assembly
def test_assemble_golden(eng, golden):
    from sgdml_b200.desc import Desc

    N = int(golden['n_atoms'])
    t = eng.GDMLTrain()
    K = t._assemble_kernel_mat(golden['R_desc'], golden['R_d_desc'], golden['tril_perms_lin'], int(golden['sig']), Desc(N))
    assert K.shape == golden['K'].shape
    assert rel_err(K, golden['K']) < 1e-12
    assert rel_err(K, K.T) < 1e-13  # symmetric


def test_assemble_col_subsets(eng, golden):
    from sgdml_b200.desc import Desc

    N = int(golden['n_atoms'])
    n = golden['K'].shape[0]
    t = eng.GDMLTrain()
    args = (golden['R_desc'], golden['R_d_desc'], golden['tril_perms_lin'], int(golden['sig']), Desc(N))
    K = t._assemble_kernel_mat(*args, col_idxs=np.s_[: 2 * 3 * N])  # block-boundary slice (train.py:1357-1374)
    assert rel_err(K, golden['K'][:, : 6 * N]) < 1e-12
    cols = np.unique(np.random.default_rng(0).integers(0, n, size=23))  # index list (train.py:1376-1407)
    K = t._assemble_kernel_mat(*args, col_idxs=cols, alloc_extra_rows=5)
    assert K.shape == (n + 5, len(cols))
    assert rel_err(K[:n], golden['K'][:, cols]) < 1e-12


@pytest.mark.parametrize('N,M,rot,swap,sig', [(3, 4, 1, 0, 5), (7, 9, 1, 1, 15), (10, 5, 2, 1, 20), (34, 3, 1, 1, 40), (42, 2, 2, 0, 50)])
def test_assemble_vs_oracle(eng, N, M, rot, swap, sig):
    from sgdml_b200 import synth
    from sgdml_b200.desc import Desc

    perms = synth.rotor_swap_group(N, rot, swap)
    R = synth.geometries(N, M, 2).reshape(M, -1)
    x, g = odesc.from_R(R)
    lin = odesc.tril_perms_lin(perms)
    K_ref = oassemble.assemble(x, g, lin, sig)
    K = eng.GDMLTrain()._assemble_kernel_mat(x, g, lin, sig, Desc(N))
    assert rel_err(K, K_ref) < 1e-12


def test_assemble_large_kernel_matches_small(eng, golden):
    """The large-molecule kernel (tables in global memory) keeps the summation order of the
    shared-memory kernel: bit-identical blocks on the golden cases."""
    from sgdml_b200 import _lib
    from sgdml_b200.desc import Desc

    N = int(golden['n_atoms'])
    n = golden['K'].shape[0]
    t = eng.GDMLTrain()
    args = (golden['R_desc'], golden['R_d_desc'], golden['tril_perms_lin'], int(golden['sig']), Desc(N))
    cols = np.unique(np.random.default_rng(1).integers(0, n, size=31))
    K_default_cols = t._assemble_kernel_mat(*args, col_idxs=cols)  # default small-molecule kernel (k_assemble_v4 here)
    _lib.lib().sgdml_b200_set_assemble_variant(2)  # the per-permutation kernel whose summation order the large one keeps
    try:
        K_small_full = t._assemble_kernel_mat(*args)
        K_small_cols = t._assemble_kernel_mat(*args, col_idxs=cols)
    finally:
        _lib.lib().sgdml_b200_set_assemble_variant(0)
    assert rel_err(K_default_cols, K_small_cols) < 1e-13
    _lib.lib().sgdml_b200_set_assemble_variant(1)
    try:
        K_full = t._assemble_kernel_mat(*args)
        K_cols = t._assemble_kernel_mat(*args, col_idxs=cols)
    finally:
        _lib.lib().sgdml_b200_set_assemble_variant(0)
    assert np.array_equal(K_cols, K_small_cols)
    assert rel_err(K_full, golden['K']) < 1e-12
    iu = np.triu_indices(n)  # the symmetric kernel computes the upper block triangle and mirrors it
    blk = (iu[0] // (3 * N)) <= (iu[1] // (3 * N))
    assert np.array_equal(K_full[iu][blk], K_small_full[iu][blk])


@pytest.mark.parametrize('variant', [0, 1])
@pytest.mark.parametrize('N,M,rot,swap,sig', [(60, 3, 1, 1, 50), (100, 2, 2, 0, 50), (53, 2, 0, 1, 30), (64, 2, 2, 1, 40)])
def test_assemble_large_molecules_vs_oracle(eng, N, M, rot, swap, sig, variant):
    """BASELINE configs 4-5 sizes (60 and 100 atoms): expanded pair tables beyond shared memory.  variant 0: the default
    routing (k_assemble_v5, compressed pair arrays on chip, up to N = 70...82 depending on S -- 76 at S = 6, 82 at
    S = 1; above that k_assemble_large, whose delta table stays in shared memory up to N = 113, so at N = 100 too),
    variant 1: the large-molecule kernel (other tables in global memory) for every size."""
    from sgdml_b200 import _lib, synth
    from sgdml_b200.desc import Desc

    perms = synth.rotor_swap_group(N, rot, swap)
    R = synth.geometries(N, M, 2).reshape(M, -1)
    x, g = odesc.from_R(R)
    lin = odesc.tril_perms_lin(perms)
    K_ref = oassemble.assemble(x, g, lin, sig)
    t = eng.GDMLTrain()
    _lib.lib().sgdml_b200_set_assemble_variant(variant)
    try:
        K = t._assemble_kernel_mat(x, g, lin, sig, Desc(N))
        assert rel_err(K, K_ref) < 1e-12
        cols = np.unique(np.random.default_rng(2).integers(0, K_ref.shape[0], size=40))
        K = t._assemble_kernel_mat(x, g, lin, sig, Desc(N), col_idxs=cols)
        assert rel_err(K, K_ref[:, cols]) < 1e-12
        Kr, nc = t._assemble_kernel_mat_device(x, g, lin, sig, col_idxs=cols, rows=(1, M))
        assert rel_err(Kr[:, :nc].cpu().numpy(), K_ref[3 * N :, cols]) < 1e-12
    finally:
        _lib.lib().sgdml_b200_set_assemble_variant(0)


@pytest.mark.parametrize('large', [0, 1])
def test_assemble_row_ranges(eng, golden, large):
    """Row-sharded assembly (sgdml_b200_assemble_rows): the block rows of any range of training
    points equal the corresponding rows of the full matrix."""
    from sgdml_b200 import _lib

    N, M = int(golden['n_atoms']), golden['R_desc'].shape[0]
    n = golden['K'].shape[0]
    t = eng.GDMLTrain()
    args = (golden['R_desc'], golden['R_d_desc'], golden['tril_perms_lin'], int(golden['sig']))
    cols = np.unique(np.random.default_rng(3).integers(0, n, size=29))
    _lib.lib().sgdml_b200_set_assemble_variant(large)
    try:
        K_cols, _ = t._assemble_kernel_mat_device(*args, col_idxs=cols)
        for lo, hi in [(0, 1), (1, M), (M // 3, 2 * M // 3 + 1)]:
            Kr, nc = t._assemble_kernel_mat_device(*args, col_idxs=cols, rows=(lo, hi))
            assert Kr.shape[0] == (hi - lo) * 3 * N
            assert np.array_equal(Kr[:, :nc].cpu().numpy(), K_cols[lo * 3 * N : hi * 3 * N, :nc].cpu().numpy())
            Kr, nc = t._assemble_kernel_mat_device(*args, rows=(lo, hi))  # all columns, part of the rows
            assert rel_err(Kr[:, :nc].cpu().numpy(), golden['K'][lo * 3 * N : hi * 3 * N]) < 1e-12
    finally:
        _lib.lib().sgdml_b200_set_assemble_variant(0)


def test_assemble_multi_launch_row_chunks(eng, golden):
    """Row ranges above the grid limit (65535 row points) run as several launches with their own first row point
    and K row offset; the test hook lowers the limit to 3 row points so that a small fixture takes that path
    (full matrix -- symmetric mode switched off -- and a column subset)."""
    from sgdml_b200 import _lib

    n = golden['K'].shape[0]
    t = eng.GDMLTrain()
    args = (golden['R_desc'], golden['R_d_desc'], golden['tril_perms_lin'], int(golden['sig']))
    cols = np.unique(np.random.default_rng(5).integers(0, n, size=31))
    K_ref, _ = t._assemble_kernel_mat_device(*args)
    Kc_ref, nc = t._assemble_kernel_mat_device(*args, col_idxs=cols)
    _lib.lib().sgdml_b200_set_assemble_variant(1003)
    try:
        K, _ = t._assemble_kernel_mat_device(*args)
        Kc, _ = t._assemble_kernel_mat_device(*args, col_idxs=cols)
    finally:
        _lib.lib().sgdml_b200_set_assemble_variant(1000 + 65535)
    assert rel_err(K[:, :n].cpu().numpy(), golden['K']) < 1e-12
    assert rel_err(K[:, :n].cpu().numpy(), K_ref[:, :n].cpu().numpy()) < 1e-14  # mirrored vs directly computed blocks
    assert np.array_equal(Kc[:, :nc].cpu().numpy(), Kc_ref[:, :nc].cpu().numpy())


def test_predict_rejects_bad_out_buffers(eng, golden):
    """Output buffers reach the engine as raw double*: wrong dtype / shape / device must raise, not corrupt memory."""
    import torch

    p = eng.GDMLPredict(golden_model(golden))
    R = golden['R_query']
    B, dim_i = R.shape
    with pytest.raises(ValueError):
        p.predict(R, out=(np.empty(B, dtype=np.float32), np.empty((B, dim_i))))
    with pytest.raises(ValueError):
        p.predict(R, out=(np.empty(B), np.empty((B, dim_i), dtype=np.float32)))
    with pytest.raises(ValueError):
        p.predict(R, out=(np.empty(B), np.empty((B + 1, dim_i))))
    with pytest.raises(ValueError):
        p.predict(torch.from_numpy(R).cuda(), out=(np.empty(B), np.empty((B, dim_i))))
    with pytest.raises(ValueError):
        p.predict(R, out=(torch.empty(B, dtype=torch.float64, device='cuda'), torch.empty((B, dim_i), dtype=torch.float64, device='cuda')))
    E, F = np.full(B, np.nan), np.empty((B, dim_i))
    (F2,) = p.predict(R, return_E=False, out=(E, F))  # E is not written when no energies are asked for
    assert F2 is F and np.all(np.isnan(E)) and rel_err(F, golden['F_query']) < 1e-10


def test_c60_icosahedral_config(eng):
    """BASELINE config 5 shape: buckyball, 60 atoms, the 120 permutations of I_h (reduced M)."""
    from sgdml_b200 import synth
    from sgdml_b200.desc import Desc

    perms, r0 = synth.config_perms_and_r0('c60')
    assert perms.shape == (120, 60)
    M = 3
    R = synth.geometries(60, M, 0, r0=r0).reshape(M, -1)
    x, g = odesc.from_R(R)
    lin = odesc.tril_perms_lin(perms)
    assert np.array_equal(eng.desc.tril_perms_lin(perms), lin)
    cols = np.arange(180, 360)  # the block column of training point 1
    K_ref = oassemble.assemble(x, g, lin, 50, col_idxs=cols)
    K = eng.GDMLTrain()._assemble_kernel_mat(x, g, lin, 50, Desc(60), col_idxs=cols)
    assert rel_err(K, K_ref) < 1e-12
    model = synth.random_model(60, 5, perms, 50, seed=4, r0=r0)
    Rq = synth.geometries(60, 7, 1, r0=r0).reshape(7, -1)
    E_ref, F_ref = opredict.Predictor(model).predict(Rq)
    E, F = eng.GDMLPredict(model).predict(Rq)
    assert rel_err(F, F_ref) < 1e-9 and rel_err(E, E_ref) < 1e-9


def test_c60_reference_fixture(eng):
    """The engine against the reference's own C60 / I_h outputs (tests/golden/big_c60_m2_s120.npz):
    k_assemble_large and the GEMM-composed large-descriptor predictor."""
    from sgdml_b200.desc import Desc

    g = load_golden('big_c60_m2_s120')
    N = int(g['n_atoms'])
    assert np.array_equal(eng.desc.tril_perms_lin(g['perms']), g['tril_perms_lin'])
    x, gd = Desc(N).from_R(g['R_train'].reshape(len(g['R_train']), -1))
    assert rel_err(x, g['R_desc']) < 1e-13 and rel_err(gd, g['R_d_desc']) < 1e-13
    c0 = int(g['col_start'])
    cols = np.arange(c0, c0 + 3 * N)
    K = eng.GDMLTrain()._assemble_kernel_mat(g['R_desc'], g['R_d_desc'], g['tril_perms_lin'], int(g['sig']), Desc(N), col_idxs=cols)
    assert rel_err(K, g['K_cols']) < 1e-11
    E, F = eng.GDMLPredict(golden_model(g)).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 1e-9 and rel_err(E, g['E_query']) < 1e-9


def test_n100_reference_fixture(eng):
    """The engine against the reference's own outputs for a 100-atom molecule (config 4 shape,
    tests/golden/big_n100_m2_s12.npz): k_assemble_large with an index-list column subset and the
    GEMM-composed predictor at D = 4950."""
    from sgdml_b200.desc import Desc

    g = load_golden('big_n100_m2_s12')
    N = int(g['n_atoms'])
    assert np.array_equal(eng.desc.tril_perms_lin(g['perms']), g['tril_perms_lin'])
    x, gd = Desc(N).from_R(g['R_train'].reshape(len(g['R_train']), -1))
    assert rel_err(x, g['R_desc']) < 1e-13 and rel_err(gd, g['R_d_desc']) < 1e-13
    K = eng.GDMLTrain()._assemble_kernel_mat(g['R_desc'], g['R_d_desc'], g['tril_perms_lin'], int(g['sig']), Desc(N), col_idxs=g['cols'])
    assert rel_err(K, g['K_cols']) < 1e-11
    E, F = eng.GDMLPredict(golden_model(g)).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 1e-9 and rel_err(E, g['E_query']) < 1e-9


# --------------------------------------------------------------------------- dense solve
_ERR_ARG = -1000  # SGDML_B200_ERR_ARG (include/sgdml_b200.h)


def _set_gemm_variant(L, variant):
    """GEMM kernel hook: 0 cp.async tiles, 2 scalar kernel, 3 TMA tiles (default).  Variant 1 selected 128x64 tiles,
    which are removed: the hook rejects it and keeps the kernel selected before, so such a case runs the default."""
    assert L.sgdml_b200_set_gemm_variant(variant) == (_ERR_ARG if variant == 1 else 0)


@pytest.mark.parametrize('variant', [0, 1, 2, 3])
@pytest.mark.parametrize('m,n,k', [(128, 128, 128), (300, 200, 64), (257, 129, 130), (64, 1000, 16), (33, 17, 7)])
def test_dgemm_nt(eng, variant, m, n, k):
    from sgdml_b200 import _lib

    L = _lib.lib()
    rng = np.random.default_rng(m + n + k)
    A = rng.standard_normal((m, k))
    B = rng.standard_normal((n, k))
    C = rng.standard_normal((m, n))
    ref = 0.75 * A @ B.T - 1.25 * C
    _set_gemm_variant(L, variant)
    try:
        _lib.check(L.sgdml_b200_dgemm_nt(m, n, k, 0.75, _lib.ptr(A), k, _lib.ptr(B), k, -1.25, _lib.ptr(C), n, None), 'dgemm')
    finally:
        L.sgdml_b200_set_gemm_variant(3)
    assert rel_err(C, ref) < 1e-13


@pytest.mark.parametrize('layout', ['lda_padded', 'offset', 'beta0_nan'])
@pytest.mark.parametrize('variant', [0, 1, 2, 3])
@pytest.mark.parametrize('m,n,k', [(128, 128, 128), (300, 200, 64), (257, 129, 130), (64, 1000, 16), (33, 17, 7)])
def test_dgemm_nt_device_layouts(eng, variant, m, n, k, layout):
    """test_dgemm_nt on device operands.  layout: padded row strides with NaN in every padding column (read by
    no kernel, C's not written); A one double off 16-byte alignment (the scalar fallback kernel); beta = 0 with
    NaN in C (C must not be read)."""
    import torch
    from sgdml_b200 import _lib

    L = _lib.lib()
    rng = np.random.default_rng(m + n + k)
    A = rng.standard_normal((m, k))
    B = rng.standard_normal((n, k))
    C = rng.standard_normal((m, n))
    alpha, beta = 0.75, (0.0 if layout == 'beta0_nan' else -1.25)
    ref = alpha * A @ B.T + beta * C
    pad = 2 if layout == 'lda_padded' else 0
    lda, ldb, ldc = k + pad, k + 2 * pad, n + pad
    nan = float('nan')
    off = 1 if layout == 'offset' else 0
    Ad = torch.full((m * lda + 1,), nan, dtype=torch.float64, device='cuda')
    Ad[off : off + m * lda].view(m, lda)[:, :k] = torch.from_numpy(A).cuda()
    Bd = torch.full((n, ldb), nan, dtype=torch.float64, device='cuda')
    Bd[:, :k] = torch.from_numpy(B).cuda()
    Cd = torch.full((m, ldc), nan, dtype=torch.float64, device='cuda')
    if layout != 'beta0_nan':
        Cd[:, :n] = torch.from_numpy(C).cuda()
    _set_gemm_variant(L, variant)
    try:
        _lib.check(
            L.sgdml_b200_dgemm_nt(
                m, n, k, alpha, Ad.data_ptr() + 8 * off, lda, Bd.data_ptr(), ldb, beta, Cd.data_ptr(), ldc, _lib.current_stream()
            ),
            'dgemm',
        )
        torch.cuda.synchronize()
    finally:
        L.sgdml_b200_set_gemm_variant(3)
    Ch = Cd.cpu().numpy()
    assert np.isnan(Ch[:, n:]).all()  # padding columns of C not written
    assert rel_err(Ch[:, :n], ref) < 1e-13


@pytest.mark.parametrize('variant', [0, 1, 3])
@pytest.mark.parametrize('n', [64, 128, 200, 513, 1400])
def test_potrf_potrs(eng, variant, n):
    import scipy.linalg
    from sgdml_b200 import _lib

    L = _lib.lib()
    rng = np.random.default_rng(n)
    X = rng.standard_normal((n, n + 20))
    A = X @ X.T + 1e-3 * np.eye(n)
    b = rng.standard_normal((n, 3))
    Af = A.copy()
    _set_gemm_variant(L, variant)
    try:
        _lib.check(L.sgdml_b200_potrf(_lib.ptr(Af), n, n, None), 'potrf')
    finally:
        L.sgdml_b200_set_gemm_variant(3)
    Lg = np.tril(Af)
    Lr = scipy.linalg.cholesky(A, lower=True)
    assert rel_err(Lg, Lr) < 1e-10
    assert rel_err(Lg @ Lg.T, A) < 1e-13
    x = b.copy()
    _lib.check(L.sgdml_b200_potrs(_lib.ptr(Af), n, n, _lib.ptr(x), 3, 3, None), 'potrs')
    assert rel_err(A @ x, b) < 1e-9
    x1 = np.ascontiguousarray(b[:, 0])
    _lib.check(L.sgdml_b200_potrs(_lib.ptr(Af), n, n, _lib.ptr(x1), 1, 1, None), 'potrs')
    assert rel_err(x1, x[:, 0]) < 1e-12


def _potrf_potrs_vs_lapack(n, lda, oz_slices, monkeypatch):
    """potrf + potrs on a device buffer of row stride lda whose strictly upper triangle and padding columns hold
    NaN, against scipy's LAPACK dpotrf / dpotrs (analytic.py:94-99): neither canary may reach L or x, and the
    padding columns must not be written."""
    import scipy.linalg
    import torch
    from sgdml_b200 import _lib

    L = _lib.lib()
    rng = np.random.default_rng(7)
    X = rng.standard_normal((n, 64))
    d = rng.uniform(0.5, 2.0, size=n)
    A = X @ X.T  # rank 64 + a positive diagonal: condition ~1e5, cheap to build
    A[np.diag_indices(n)] += d
    b = rng.standard_normal((n, 2))
    c, low = scipy.linalg.cho_factor(A, lower=True, check_finite=False)
    x_ref = scipy.linalg.cho_solve((c, low), b, check_finite=False)
    if oz_slices:
        monkeypatch.setenv('SGDML_B200_OZAKI_SLICES', str(oz_slices))
    Ad = torch.full((n, lda), float('nan'), dtype=torch.float64, device='cuda')
    Ad[:, :n] = torch.from_numpy(A).cuda().tril_() + Ad.new_full((n, n), float('nan')).triu_(1)
    _lib.check(L.sgdml_b200_potrf(Ad.data_ptr(), n, lda, _lib.current_stream()), 'potrf')
    xd = torch.from_numpy(b.copy()).cuda()
    _lib.check(L.sgdml_b200_potrs(Ad.data_ptr(), n, lda, xd.data_ptr(), 2, 2, _lib.current_stream()), 'potrs')
    torch.cuda.synchronize()
    if lda > n:
        assert bool(torch.isnan(Ad[:, n:]).all())
    Lg = np.tril(Ad[:, :n].cpu().numpy())
    tol = 1e-11 if not oz_slices else 1e-9
    assert rel_err(Lg, np.tril(c)) < tol
    x = xd.cpu().numpy()
    assert rel_err(x, x_ref) < tol * 10
    assert rel_err(A @ x, b) < tol * 10


@pytest.mark.parametrize('oz_slices', [0, 7])
def test_potrf_potrs_large_outer_block(eng, oz_slices, monkeypatch):
    """n >= 16384 takes the NBO = 1024 outer blocking and the triangular super-tile order of the trailing GEMM --
    the configuration BASELINE config 2 (n = 63000) runs -- against scipy's LAPACK dpotrf / dpotrs
    (analytic.py:94-99).  oz_slices = 7: the same factorisation with the int8 (wgmma) trailing updates.
    n = 16500 is not a multiple of any block size."""
    _potrf_potrs_vs_lapack(16500, 16500, oz_slices, monkeypatch)


@pytest.mark.parametrize('oz_slices', [0, 7])
def test_potrf_potrs_large_outer_block_padded_stride(eng, oz_slices, monkeypatch):
    """The NBO = 1024 path with the padded stride lda = n + 1 of the analytic solver, ending in a one-column
    block: n = 16385 = 16 * 1024 + 1."""
    _potrf_potrs_vs_lapack(16385, 16386, oz_slices, monkeypatch)


def test_train_analytic_large_outer_block_residual(eng):
    """Aspirin shape at M = 270 (n = 17010 >= 16384: NBO = 1024 path) through GDMLTrain.train, checked by the
    K.v identity: (K - lam I) alphas reproduces the labels through the predictor kernels, which share no code with
    the assembly and Cholesky kernels (sgdml_b200/diagnostics.py; analytic.py:65-99)."""
    from sgdml_b200 import synth
    from sgdml_b200.diagnostics import residual_report

    from sgdml_b200 import _lib

    task = synth.make_config_task('aspirin', n_train=270)
    models = {}
    for slices, tol in ((-1, 1e-9), (0, 1e-12)):  # default (int8-sliced trailing updates at this size) and all-FP64
        _lib.lib().sgdml_b200_set_solve_slices(slices)
        try:
            model = eng.GDMLTrain().train(task)
        finally:
            _lib.lib().sgdml_b200_set_solve_slices(-1)
        assert model['solver_name'] == 'analytic'
        rep = residual_report(model, task)
        assert rep['residual_rel'] < tol, rep
        assert rep['force_rel_max_train'] < 1e-4, rep
        models[slices] = model
    # the two factorisations give the same force field far inside the 1e-6 bound of north_star
    Rq = synth.geometries(21, 32, 1).reshape(32, -1)
    _, F_a = eng.GDMLPredict(models[-1]).predict(Rq)
    _, F_b = eng.GDMLPredict(models[0]).predict(Rq)
    assert rel_err(F_a, F_b) < 1e-8


def test_potrf_not_positive_definite(eng):
    from sgdml_b200 import _lib

    n = 300
    rng = np.random.default_rng(0)
    X = rng.standard_normal((n, n))
    A = X @ X.T + np.eye(n)
    A[170, 170] = -1.0  # leading minor of order 171 fails
    Af = A.copy()  # (keep a reference: the engine reads the buffer behind the raw pointer)
    rc = _lib.lib().sgdml_b200_potrf(_lib.ptr(Af), n, n, None)
    assert rc == 171
    with pytest.raises(np.linalg.LinAlgError, match='not positive definite'):
        _lib.check(rc, 'potrf')


def test_solve_analytic_golden(eng, golden):
    """alphas = -(-K + lam I)^-1 y (analytic.py:65-99) from the reference's own K."""
    from sgdml_b200 import _lib

    task = golden_task(golden)
    y, _, _ = otrain.labels(task)
    n = golden['K'].shape[0]
    Kneg = -golden['K'].copy()
    alphas = np.empty(n)
    _lib.check(
        _lib.lib().sgdml_b200_solve_analytic(_lib.ptr(Kneg), n, n, float(golden['lam']), _lib.ptr(y), _lib.ptr(alphas), None),
        'solve_analytic',
    )
    # the system has cond ~1e11: compare the residual and the predictions, not alphas digit by digit
    A = -golden['K'] + float(golden['lam']) * np.eye(n)
    assert np.linalg.norm(A @ (-alphas) - y) < 1e-9 * np.linalg.norm(y)
    assert rel_err(alphas, golden['alphas_F']) < 1e-3


# --------------------------------------------------------------------------- end to end
def test_train_end_to_end_golden(eng, golden):
    """GDMLTrain.train(task) -> model -> GDMLPredict.predict == reference train + predict within 1e-6."""
    task = golden_task(golden)
    model = eng.GDMLTrain().train(task)
    assert np.array_equal(model['tril_perms_lin'], golden['tril_perms_lin'])
    assert model['R_desc'].shape == golden['model_R_desc'].shape  # (D, M) transposed layout
    assert rel_err(model['R_desc'], golden['model_R_desc']) < 1e-14
    assert abs(model['std'] - float(golden['std'])) < 1e-13
    assert abs(model['c'] - float(golden['c'])) < 1e-6 * max(1.0, abs(float(golden['c'])))
    p = eng.GDMLPredict(model)
    E, F = p.predict(golden['R_query'])
    assert rel_err(F, golden['F_query']) < 1e-6
    assert rel_err(E, golden['E_query']) < 1e-6


def _train_vs_oracle(eng, task):
    """Engine-trained model vs oracle-trained model, predictions on 100 query geometries within 1e-6."""
    from sgdml_b200 import synth

    model = eng.GDMLTrain().train(task)
    ref = otrain.train(task)
    Rq = synth.geometries(9, 100, 1).reshape(100, -1)
    E_ref, F_ref = opredict.Predictor(ref).predict(Rq)
    E, F = eng.GDMLPredict(model).predict(Rq)
    assert rel_err(F, F_ref) < 1e-6
    assert rel_err(E, E_ref) < 1e-6


def test_train_ethanol_config_vs_oracle(eng):
    """BASELINE config 1 (9 atoms, 200 training points, 6 perms): engine-trained model vs
    oracle-trained model, predictions on 100 query geometries within 1e-6."""
    from sgdml_b200 import synth

    _train_vs_oracle(eng, synth.make_config_task('ethanol'))


def test_train_ethanol_odd_size_padded_stride(eng):
    """The ethanol configuration at 201 training points: n = 5427 is odd, so the analytic solver assembles and
    factorises K with the padded row stride n + 1 from start to finish."""
    from sgdml_b200 import synth

    _train_vs_oracle(eng, synth.make_config_task('ethanol', n_train=201))


def test_model_npz_roundtrip(eng, golden, tmp_path):
    """The model dict survives np.savez_compressed / np.load like the reference's (cli.py:1098, io.py:404)."""
    task = golden_task(golden)
    model = eng.GDMLTrain().train(task)
    path = tmp_path / 'model.npz'
    np.savez_compressed(path, **model)
    with np.load(path, allow_pickle=True) as f:
        loaded = {k: f[k] for k in f.files}
    assert str(loaded['type']) == 'm' and loaded['R_desc'].shape == model['R_desc'].shape
    E0, F0 = eng.GDMLPredict(model).predict(golden['R_query'])
    E1, F1 = eng.GDMLPredict(loaded).predict(golden['R_query'])
    assert np.array_equal(F0, F1) and np.array_equal(E0, E1)


def test_large_descriptor_kv_and_set_alphas(eng):
    """D > 256 (GEMM-composed predictor): K @ v through set_alphas / kmatvec_train, N = 24."""
    from sgdml_b200 import synth

    N, M = 24, 6
    perms = synth.rotor_swap_group(N, 1, 1)
    model, x, g = _oracle_model(N, M, perms, 30, seed=5)
    K_ref = oassemble.assemble(x, g, model['tril_perms_lin'], 30)
    v = np.random.default_rng(2).standard_normal(M * 3 * N)
    p = eng.GDMLPredict(model)
    p.set_R_desc(x)
    p.set_R_d_desc(g)
    p.set_alphas(v)
    assert rel_err(p.kmatvec_train().ravel(), K_ref @ v) < 1e-10
    p.set_alphas(model['alphas_F'])
    E, F = p.predict()
    E_ref, F_ref = opredict.Predictor(model).predict(synth.geometries(N, M, 5).reshape(M, -1))
    assert rel_err(F, F_ref) < 1e-10 and rel_err(E, E_ref) < 1e-10


@pytest.mark.parametrize('B', [1, 2, 7, 100, 700])
def test_predict_small_batches_split_over_training_points(eng, B):
    """Small batches split the sweep over M across CTAs (per-split partial planes summed by the finishing
    kernel): same answer as the oracle for any batch size, including the single-geometry MD case."""
    from sgdml_b200 import synth

    N, M = 9, 200
    perms = synth.rotor_swap_group(N, 1, 1)
    model, _, _ = _oracle_model(N, M, perms, 20, seed=11)
    Rq = synth.geometries(N, B, 1).reshape(B, -1)
    E_ref, F_ref = opredict.Predictor(model).predict(Rq)
    E, F = eng.GDMLPredict(model).predict(Rq)
    assert rel_err(F, F_ref) < 1e-10 and rel_err(E, E_ref) < 1e-10
    N2, M2 = 21, 130
    perms2 = synth.rotor_swap_group(N2, 1, 1)
    model2, _, _ = _oracle_model(N2, M2, perms2, 20, seed=12)
    Rq2 = synth.geometries(N2, min(B, 40), 1).reshape(min(B, 40), -1)
    E_ref, F_ref = opredict.Predictor(model2).predict(Rq2)
    E, F = eng.GDMLPredict(model2).predict(Rq2)
    assert rel_err(F, F_ref) < 1e-10 and rel_err(E, E_ref) < 1e-10


# --------------------------------------------------------------------------- (f)4: lattices and energy constraints
def _pbc_ecstr_task(g):
    from sgdml_b200 import synth

    N = int(g['n_atoms'])
    t = synth.make_task(N, g['R_train'].shape[0], g['perms'], int(g['sig']), lam=float(g['lam']))
    if 'lattice' in g:
        t['lattice'] = g['lattice']
    t['use_E_cstr'] = bool(g['use_E_cstr'])
    return t


def _pbc_ecstr_model(g):
    m = golden_model(g)
    if 'lattice' in g:
        m['lattice'] = g['lattice']
    if 'alphas_E' in g:
        m['alphas_E'] = g['alphas_E']
    return m


@pytest.mark.parametrize('name', ['pbc_n6_m8', 'ecstr_n6_m8'])
def test_pbc_and_energy_constraints_vs_reference(eng, name):
    """Engine against fixtures generated by the unmodified reference with a lattice (utils/desc.py:44-77) and with
    energy constraints in the kernel (train.py:234-300, predict.py:219-229): descriptors, K (incl. the M extra rows /
    columns), predictions of the reference's model, and the engine's own training run (1e-6 rel, north_star)."""
    from sgdml_b200.desc import Desc

    g = load_golden(name)
    N, M = int(g['n_atoms']), g['R_train'].shape[0]
    d = Desc(N)
    lat_and_inv = (g['lattice'], np.linalg.inv(g['lattice'])) if 'lattice' in g else None
    x, gd = d.from_R(g['R_train'].reshape(M, -1), lat_and_inv=lat_and_inv)
    assert rel_err(x, g['R_desc']) < 1e-14 and rel_err(gd, g['R_d_desc']) < 1e-13
    t = eng.GDMLTrain()
    K = t._assemble_kernel_mat(g['R_desc'], g['R_d_desc'], g['tril_perms_lin'], int(g['sig']), d, use_E_cstr=bool(g['use_E_cstr']))
    assert K.shape == g['K'].shape and rel_err(K, g['K']) < 1e-12
    p = eng.GDMLPredict(_pbc_ecstr_model(g))
    E, F = p.predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 1e-9 and rel_err(E, g['E_query']) < 1e-9
    E, F = p.predict(g['R_train'].reshape(M, -1))
    assert rel_err(F, g['F_train_pred']) < 1e-9 and rel_err(E, g['E_train_pred']) < 1e-9
    model = t.train(_pbc_ecstr_task(g))
    assert ('alphas_E' in model) == bool(g['use_E_cstr']) and ('lattice' in model) == ('lattice' in g)
    assert abs(float(model['c']) - float(g['c'])) < 1e-6 * abs(float(g['c']))
    E2, F2 = eng.GDMLPredict(model).predict(g['R_query'])
    assert rel_err(F2, g['F_query']) < 1e-6 and rel_err(E2, g['E_query']) < 1e-6


def test_energy_constraints_large_descriptor_path(eng):
    """The energy-constraint terms in the GEMM-composed predictor (D > 256) against the oracle."""
    from sgdml_b200 import synth

    N, M = 24, 12
    perms = synth.rotor_swap_group(N, 1, 1)
    model, x, g = _oracle_model(N, M, perms, 30)
    model['alphas_E'] = np.random.default_rng(4).standard_normal(M)
    Rq = synth.geometries(N, 7, 1).reshape(7, -1)
    E, F = eng.GDMLPredict(model).predict(Rq)
    E_ref, F_ref = opredict.Predictor(model).predict(Rq)
    assert rel_err(F, F_ref) < 1e-10 and rel_err(E, E_ref) < 1e-10


# --------------------------------------------------------------------------- (f)2: residency across a sigma grid
def test_sigma_grid_reuses_descriptors_and_buffers(eng):
    """`sgdml all` retrains the same points for several length scales with one GDMLTrain instance (cli.py:802-806,
    981-1083): the engine keeps the (sigma-independent) descriptors on the device and reuses the kernel-matrix
    buffer; the models equal those of fresh, independent training runs bit for bit."""
    from sgdml_b200 import synth

    N, M = 9, 30
    perms = synth.rotor_swap_group(N, 1, 1)
    t = eng.GDMLTrain()
    models = []
    for sig in (10, 20, 30):
        models.append(t.train(synth.make_task(N, M, perms, sig)))
    assert t.cache_stats['desc_misses'] == 1 and t.cache_stats['desc_hits'] == 2
    assert t.cache_stats['K_allocated'] == 1 and t.cache_stats['K_reused'] == 2
    for sig, m in zip((10, 20, 30), models):
        fresh = eng.GDMLTrain().train(synth.make_task(N, M, perms, sig))
        assert np.array_equal(m['alphas_F'], fresh['alphas_F']) and float(m['c']) == float(fresh['c'])
    # a different training set is a cache miss, and release_buffers() empties everything
    t.train(synth.make_task(N, M, perms, 20, seed=3))
    assert t.cache_stats['desc_misses'] == 2
    t.release_buffers()
    assert not t._desc_cache and t._K_buf is None


def test_ase_calculator_core_units(eng, golden):
    """intf/ase_calc.py:81-110 without ASE: positions in Angstrom -> energy in eV, forces (N, 3) in eV/Ang."""
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV, SGDMLCalculatorCore

    calc = SGDMLCalculatorCore()
    calc._setup(golden_model(golden), _KCAL_PER_MOL_IN_EV, _KCAL_PER_MOL_IN_EV)
    N = int(golden['n_atoms'])
    res = calc.compute(golden['R_query'][0].reshape(N, 3))
    assert res['forces'].shape == (N, 3)
    assert rel_err(res['forces'].ravel(), golden['F_query'][0] * _KCAL_PER_MOL_IN_EV) < 1e-10
    assert rel_err(res['energy'], golden['E_query'][:1] * _KCAL_PER_MOL_IN_EV) < 1e-10
    assert abs(_KCAL_PER_MOL_IN_EV - 0.0433641) < 1e-6


# --------------------------------------------------------------------------- small-molecule assembly kernels
@pytest.mark.parametrize('variant', [2, 3, 4, 5])
def test_assemble_v3_kernel(eng, golden, variant):
    """k_assemble_v4 (permutation chunks, delta on the fly, resident row tables, byte permutation tables, odd table
    strides, type-major phase A over kept column atoms), k_assemble_v5 (the same on the compressed pair arrays) and
    k_assemble (per-permutation phases, the kernel they are compared with elsewhere) against the reference's K: full
    matrix (symmetric mode), a column subset, row ranges, and the multi-launch row path.  Variant 3 selected
    k_assemble_v3, which is removed: the hook rejects it and keeps the default routing."""
    from sgdml_b200 import _lib

    N, M = int(golden['n_atoms']), golden['R_desc'].shape[0]
    n = golden['K'].shape[0]
    t = eng.GDMLTrain()
    args = (golden['R_desc'], golden['R_d_desc'], golden['tril_perms_lin'], int(golden['sig']))
    cols = np.unique(np.random.default_rng(11).integers(0, n, size=37))
    L = _lib.lib()
    assert L.sgdml_b200_set_assemble_variant(variant) == (_ERR_ARG if variant == 3 else 0)
    try:
        K, _ = t._assemble_kernel_mat_device(*args)
        assert rel_err(K[:, :n].cpu().numpy(), golden['K']) < 1e-12
        Kc, nc = t._assemble_kernel_mat_device(*args, col_idxs=cols)
        assert rel_err(Kc[:, :nc].cpu().numpy(), golden['K'][:, cols]) < 1e-12
        lo, hi = M // 3, 2 * M // 3 + 1
        Kr, nc = t._assemble_kernel_mat_device(*args, col_idxs=cols, rows=(lo, hi))
        assert rel_err(Kr[:, :nc].cpu().numpy(), golden['K'][lo * 3 * N : hi * 3 * N][:, cols]) < 1e-12
        L.sgdml_b200_set_assemble_variant(1002)
        K2, _ = t._assemble_kernel_mat_device(*args)
        assert rel_err(K2[:, :n].cpu().numpy(), golden['K']) < 1e-12
    finally:
        L.sgdml_b200_set_assemble_variant(1000 + 65535)
        L.sgdml_b200_set_assemble_variant(0)


def test_assemble_v3_many_permutations(eng):
    """A permutation group too large for one chunk (S = 81, 12 atoms... PG < S) and a mid-sized molecule whose sub-blocks
    are split over grid.z (N = 36): v4 and v5 against the per-permutation kernel, full matrix and a column subset."""
    from sgdml_b200 import _lib, synth
    from sgdml_b200.desc import Desc, tril_perms_lin

    L = _lib.lib()
    t = eng.GDMLTrain()
    for N, M, rot, swap in ((13, 5, 4, 0), (36, 4, 3, 1)):
        perms = synth.rotor_swap_group(N, rot, swap)
        R = synth.geometries(N, M, 0).reshape(M, -1)
        x, g = Desc(N).from_R(R)
        lin = tril_perms_lin(perms)
        out, sub = {}, {}
        cols = np.unique(np.random.default_rng(N).integers(0, 3 * N * M, size=3 * M))
        for v in (2, 4, 5):
            L.sgdml_b200_set_assemble_variant(v)
            try:
                K, nc = t._assemble_kernel_mat_device(x, g, lin, 25)
                out[v] = K[:, :nc].cpu().numpy()
                Kc, ncc = t._assemble_kernel_mat_device(x, g, lin, 25, col_idxs=cols)
                sub[v] = Kc[:, :ncc].cpu().numpy()
            finally:
                L.sgdml_b200_set_assemble_variant(0)
        for v in (4, 5):
            assert rel_err(out[v], out[2]) < 1e-12
            assert rel_err(out[v], out[v].T) < 1e-12  # the mirrored blocks
            assert rel_err(sub[v], out[2][:, cols]) < 1e-12 and rel_err(sub[2], out[2][:, cols]) < 1e-12


# --------------------------------------------------------------------------- (f)3: MD latency path (graph replay)
@pytest.mark.parametrize('zero_copy', ['1', '0'])
def test_small_batch_graph_replay(eng, golden, monkeypatch, zero_copy):
    """Host-buffer batches of <= 16 geometries replay a captured CUDA graph (csrc/predict.cu predict_graph): same
    results as plain launches, across batch sizes, repeated calls, new coefficients (set_alphas keeps the graph valid)
    and with / without the energy output.  zero_copy: three kernel nodes reading / writing pinned host memory directly
    (k_desc_query_rows; the default) vs copy nodes around the four kernels of the large-batch path."""
    from sgdml_b200.desc import Desc

    monkeypatch.setenv('SGDML_B200_GRAPH_ZEROCOPY', zero_copy)

    model = golden_model(golden)
    N, M = int(golden['n_atoms']), golden['R_train'].shape[0]
    p = eng.GDMLPredict(model)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    ref = {B: p.predict(golden['R_query'][:B]) for B in (1, 3)}
    monkeypatch.setenv('SGDML_B200_GRAPH', '1')
    for rep in range(3):  # first call captures, later calls replay
        for B in (1, 3):
            E, F = p.predict(golden['R_query'][:B])
            assert np.array_equal(F, ref[B][1]) and np.array_equal(E, ref[B][0])
    (F1,) = p.predict(golden['R_query'][:1], return_E=False)
    assert np.array_equal(F1, ref[1][1])
    E, F = p.predict(golden['R_query'][1])  # a different geometry through the replayed graph
    assert rel_err(F[0], golden['F_query'][1]) < 1e-10 and rel_err(E, golden['E_query'][1:2]) < 1e-10
    # new coefficients through the same handle: the graph reads the updated device arrays
    _, gd = Desc(N).from_R(golden['R_train'].reshape(M, -1))
    p.set_R_d_desc(gd)
    p.set_alphas(2.0 * golden['alphas_F'])
    E2, F2 = p.predict(golden['R_query'][:1])
    assert rel_err(F2, 2.0 * golden['F_query'][:1]) < 1e-10


# --------------------------------------------------------------------------- device-block cache of the predictor
def test_predictor_block_cache_reuse(eng, golden):
    """Model arrays and workspaces of a destroyed predictor are kept for the next one of the same shape
    (csrc/core.cu cached_malloc / cached_free).  Destroying a predictor whose kernels are still in flight (CUDA tensors
    in and out: nothing synchronises), creating another one on the recycled blocks with DIFFERENT coefficients and
    predicting again must give each model's own results; releasing the cache in between changes nothing."""
    import torch

    from sgdml_b200 import _lib

    model = golden_model(golden)
    model2 = dict(model)
    model2['R_d_desc_alpha'] = 3.0 * np.asarray(model['R_d_desc_alpha'])
    Rq = np.repeat(golden['R_query'], 200, axis=0)
    Rd = torch.from_numpy(Rq).cuda()
    ref = eng.GDMLPredict(model).predict(golden['R_query'])[1]
    for rep in range(4):
        p = eng.GDMLPredict(model)
        E1, F1 = p.predict(Rd)  # asynchronous: outputs are CUDA tensors
        del p  # blocks go back to the cache while the kernels may still run
        p2 = eng.GDMLPredict(model2)  # same shapes: recycled blocks
        E2, F2 = p2.predict(Rd)
        torch.cuda.synchronize()
        n = golden['R_query'].shape[0]
        assert rel_err(F1.cpu().numpy()[::200][:n], ref) < 1e-12
        assert rel_err(F2.cpu().numpy()[::200][:n], 3.0 * ref) < 1e-12
        del p2
        if rep == 1:
            assert _lib.lib().sgdml_b200_release_workspaces() == 0
