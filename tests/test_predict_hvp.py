"""Hessian-vector products: sgdml_b200_predict_hvp / GDMLPredict.predict_hvp, HV = (dF/dR) V = -H V per geometry.

CPU: the torch oracle (tests/hvp_oracle.py) against oracle.predict.Predictor, its HV against central differences of its
own F, and the NumPy model of the engine's GEMM-form HVP against the oracle, including training geometries, where the
floor under n in k_transform_tangent_rows is what keeps the result finite and right.
GPU: the engine against the oracle on every golden model (D <= 256 on the fused predictor's models, D > 256, S = 120 and
240 atoms), at training geometries against central differences of its own F, symmetry, chunking, refreshed
coefficients, NumPy / CUDA / pinned I/O and argument errors, and `predict` unchanged by an HVP.  Bounds are max-abs
error over max-abs reference."""

import contextlib

import numpy as np
import pytest

import hvp_oracle as ho
import predict_checks as pc
from conftest import rel_err
from oracle import desc as odesc
from oracle import predict as opredict

ALL = ho.FIXTURES + ['big_c60_m2_s120', 'big_n240_m2_s3']


def _rng_v(R, seed):
    return np.random.default_rng(seed).standard_normal(np.shape(R))


# --------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('name', ALL)
def test_torch_oracle_matches_predictor(name):
    """E and F of the torch restatement equal oracle.predict.Predictor within 1e-12 of the largest term magnitude
    (predict_checks.predict_abs_scale).  On the well-conditioned fixtures that is 1e-12 of max |F| itself; pbc_n6_m8 and
    ecstr_n6_m8 cancel terms ~50x larger than their outputs, so another summation order moves them further."""
    model, Rq, _ = ho.fixture_model(name)
    op = opredict.Predictor(model)
    E0, F0 = op.predict(Rq)
    E1, F1 = ho.TorchOracle(model).ef_np(Rq)
    sE, sF = pc.predict_abs_scale(model, Rq, oracle=op)
    assert np.max(np.abs(F1 - F0)) <= 1e-12 * np.max(sF), rel_err(F1, F0)
    assert np.max(np.abs(E1 - E0)) <= 1e-12 * np.max(sE), rel_err(E1, E0)
    if name not in ('pbc_n6_m8', 'ecstr_n6_m8'):
        assert rel_err(F1, F0) <= 1e-12 and rel_err(E1, E0) <= 1e-12


@pytest.mark.parametrize('name', ALL)
def test_oracle_hvp_matches_central_differences(name):
    model, Rq, _ = ho.fixture_model(name)
    to = ho.TorchOracle(model)
    R = Rq[:3]
    V = _rng_v(R, 1)
    fd = ho.central_diff_hvp(lambda r: to.ef_np(r)[1], R, V)
    assert rel_err(to.hvp(R, V), fd) <= 1e-6


@pytest.mark.parametrize('name', ALL)
def test_gemm_form_model_matches_oracle(name):
    model, Rq, _ = ho.fixture_model(name)
    R = Rq[:3]
    V = _rng_v(R, 2)
    assert rel_err(ho.gemm_form_hvp(model, R, V), ho.TorchOracle(model).hvp(R, V)) <= 1e-10


@pytest.mark.parametrize('name', ALL)
def test_gemm_form_model_at_training_geometries(name):
    """delta = 0 exactly for one (training point, permutation) pair: the GEMM-form x5, a and ds are rounding noise there,
    and the floor under n keeps a ds / n at its true limit 0."""
    model, _, Rt = ho.fixture_model(name)
    to = ho.TorchOracle(model)
    R = Rt[:3]
    V = _rng_v(R, 3)
    HV = ho.gemm_form_hvp(model, R, V)
    assert np.all(np.isfinite(HV))
    assert rel_err(HV, ho.central_diff_hvp(lambda r: to.ef_np(r)[1], R, V)) <= 1e-6


def test_gemm_form_model_fails_at_training_geometries_without_the_floor():
    """The floor is load-bearing: without it the same training geometries are non-finite or far off on these models."""
    failed = []
    for name in ('n9_m16_s6', 'n12_m8_s12', 'ecstr_n6_m8', 'pbc_n6_m8', 'big_c60_m2_s120', 'big_n240_m2_s3'):
        model, _, Rt = ho.fixture_model(name)
        to = ho.TorchOracle(model)
        R = Rt[:3]
        V = _rng_v(R, 3)
        HV = ho.gemm_form_hvp(model, R, V, guard=False)
        fd = ho.central_diff_hvp(lambda r: to.ef_np(r)[1], R, V)
        if not np.all(np.isfinite(HV)) or rel_err(HV, fd) > 1e-6:
            failed.append(name)
    print('\n[hvp floor] without it, wrong at training geometries of', failed)
    assert len(failed) >= 3, failed


# --------------------------------------------------------------------------- GPU
@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


@contextlib.contextmanager
def _chunk_cap(n):
    from sgdml_b200 import _lib

    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(int(n)), 'set_predict_chunk')
    try:
        yield
    finally:
        _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(0), 'set_predict_chunk')


_WORST = {}


@pytest.mark.gpu
@pytest.mark.parametrize('name', ALL)
def test_hvp_matches_oracle(eng, name):
    model, Rq, _ = ho.fixture_model(name)
    R = Rq
    V = _rng_v(R, 4)
    HV = eng.GDMLPredict(model).predict_hvp(R, V)
    err = rel_err(HV, ho.TorchOracle(model).hvp(R, V))
    _WORST[name] = err
    print('\n[hvp] %s: B = %d, max|HV - HV_oracle| / max|HV_oracle| = %.2e (worst so far %.2e)'
          % (name, R.shape[0], err, max(_WORST.values())))
    assert err <= 1e-8


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'pbc_n6_m8', 'big_n100_m2_s12'])
def test_hvp_at_training_geometries(eng, name):
    model, _, Rt = ho.fixture_model(name)
    p = eng.GDMLPredict(model)
    R = Rt[:4]
    V = _rng_v(R, 5)
    HV = p.predict_hvp(R, V)
    assert np.all(np.isfinite(HV))
    fd = ho.central_diff_hvp(lambda r: p.predict(r)[1], R, V)
    err = rel_err(HV, fd)
    print('\n[hvp] %s at training geometries: against central differences of predict %.2e' % (name, err))
    assert err <= 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'ecstr_n6_m8', 'big_n100_m2_s12'])
def test_hvp_is_symmetric(eng, name):
    model, Rq, _ = ho.fixture_model(name)
    p = eng.GDMLPredict(model)
    R = Rq[:3]
    U, V = _rng_v(R, 6), _rng_v(R, 7)
    HU, HV = p.predict_hvp(R, U), p.predict_hvp(R, V)
    lhs, rhs = np.sum(U * HV, axis=1), np.sum(V * HU, axis=1)
    scale = np.linalg.norm(U, axis=1) * np.linalg.norm(HV, axis=1)
    assert np.all(np.abs(lhs - rhs) <= 1e-10 * scale), (lhs, rhs)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12'])
def test_hvp_chunks_and_tail(eng, name):
    model, Rq, _ = ho.fixture_model(name)
    R = np.concatenate([Rq] * 4)[:10]
    V = _rng_v(R, 8)
    HV0 = eng.GDMLPredict(model).predict_hvp(R, V)
    with _chunk_cap(3):  # chunks of 3, 3, 3, 1
        HV1 = eng.GDMLPredict(model).predict_hvp(R, V)
    print('\n[hvp chunks] %s: bit-identical %s, max diff %.2e' % (name, np.array_equal(HV0, HV1), rel_err(HV1, HV0)))
    assert rel_err(HV1, HV0) <= 1e-13


@pytest.mark.gpu
def test_hvp_after_new_coefficients(eng):
    """A D <= 256 model keeps XcT / JAT after its first HVP; set_alphas must refresh them (and alphas_E be used)."""
    model, Rq, Rt = ho.fixture_model('n9_m16_s6')
    M = Rt.shape[0]
    _, gd = odesc.from_R(Rt)
    p = eng.GDMLPredict(model)
    p.set_R_d_desc(gd)
    R = Rq[:4]
    V = _rng_v(R, 9)
    assert rel_err(p.predict_hvp(R, V), ho.TorchOracle(model).hvp(R, V)) <= 1e-8
    rng = np.random.default_rng(10)
    aF = rng.standard_normal(M * Rt.shape[1])
    aE = rng.standard_normal(M)
    p.set_alphas(aF, alphas_E=aE)
    m2 = dict(model)
    m2['R_d_desc_alpha'] = odesc.d_desc_dot_vec(gd, aF.reshape(M, -1))
    m2['alphas_E'] = aE
    ref = ho.TorchOracle(m2).hvp(R, V)
    assert rel_err(ref, ho.TorchOracle(model).hvp(R, V)) > 1e-2  # the coefficients matter
    assert rel_err(p.predict_hvp(R, V), ref) <= 1e-8


@pytest.mark.gpu
def test_hvp_io_forms_and_argument_errors(eng):
    import torch

    model, Rq, _ = ho.fixture_model('n12_m8_s12')
    p = eng.GDMLPredict(model)
    R = Rq[:5]
    V = _rng_v(R, 11)
    HV = p.predict_hvp(R, V)
    assert isinstance(HV, np.ndarray) and HV.shape == R.shape
    Rd, Vd = torch.from_numpy(R).cuda(), torch.from_numpy(V).cuda()
    HVd = p.predict_hvp(Rd, Vd)
    torch.cuda.synchronize()
    assert HVd.is_cuda and np.array_equal(HVd.cpu().numpy(), HV)
    Rp, Vp = torch.from_numpy(R).pin_memory(), torch.from_numpy(V).pin_memory()
    HVp = p.predict_hvp(Rp, Vp)
    assert HVp.is_pinned() and np.array_equal(HVp.numpy(), HV)
    out = torch.full(Rd.shape, float('nan'), dtype=torch.float64, device='cuda')
    assert p.predict_hvp(Rd, Vd, out=out) is out
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), HV)
    # single geometry (3N,)
    assert np.array_equal(p.predict_hvp(R[0], V[0]), HV[:1])
    # V of the wrong shape, dtype, type or device: ValueError, nothing written
    out = np.full(R.shape, np.nan)
    for bad in (V[:4], V.astype(np.float32), Vd, V.reshape(5, -1, 3)):
        with pytest.raises(ValueError):
            p.predict_hvp(R, bad, out=out)
    assert np.all(np.isnan(out))
    outd = torch.full(Rd.shape, float('nan'), dtype=torch.float64, device='cuda')
    for bad in (Vd[:4], Vd.float(), torch.from_numpy(V)):
        with pytest.raises(ValueError):
            p.predict_hvp(Rd, bad, out=outd)
    with pytest.raises(ValueError):  # an out buffer on the wrong device
        p.predict_hvp(Rd, Vd, out=np.full(R.shape, np.nan))
    torch.cuda.synchronize()
    assert torch.isnan(outd).all()


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12'])
def test_predict_unchanged_by_hvp(eng, name):
    model, Rq, _ = ho.fixture_model(name)
    p = eng.GDMLPredict(model)
    E0, F0 = p.predict(Rq)
    E0b, F0b = p.predict(Rq[:1])  # (graph path)
    p.predict_hvp(np.concatenate([Rq] * 3), _rng_v(np.concatenate([Rq] * 3), 12))
    E1, F1 = p.predict(Rq)
    E1b, F1b = p.predict(Rq[:1])
    assert np.array_equal(E0, E1) and np.array_equal(F0, F1)
    assert np.array_equal(E0b, E1b) and np.array_equal(F0b, F1b)
