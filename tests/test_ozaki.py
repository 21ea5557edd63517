"""Bring-up harness for the wgmma FP64-via-INT8 GEMM (csrc/ozaki.cu): the split kernel and the raw int32 level sums
against the exact model tests/ozaki_model.py, and its callers (potrf's trailing update, the large-descriptor predictor
and K.v) against their FP64 forms.  The GEMM itself is tested bit for bit in every class in test_ozaki_classes.py.
GPU only."""

import numpy as np
import pytest

import ozaki_model as om
from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_debug_flags(monkeypatch):
    """SGDML_B200_OZAKI_DBG switches parts of the kernel off."""
    monkeypatch.delenv('SGDML_B200_OZAKI_DBG', raising=False)


# ------------------------------------------------------------------------------------------------
# Staged bring-up: (1) the split kernel alone, (2) the raw int32 level sums of one tile against exact
# NumPy integer products, then the GEMM classes.  Run in this order when the kernel first meets hardware:
#   pytest tests/test_ozaki.py -x -q -k "stage1 or stage2"
def _debug(m, n, k, S, seed=0, with_product=True):
    import torch

    from sgdml_b200 import _lib

    _lib.require_gpu()
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((m, k)) * np.exp2(rng.integers(-3, 3, size=(m, 1)).astype(np.float64))
    B = rng.standard_normal((n, k))
    mp, np_, kp = -(-m // 128) * 128, -(-n // 128) * 128, -(-k // 128) * 128
    Ad, Bd = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    pa = torch.zeros((S, mp, kp), dtype=torch.int8, device='cuda')
    pb = torch.zeros((S, np_, kp), dtype=torch.int8, device='cuda')
    ea = torch.zeros(mp, dtype=torch.int32, device='cuda')
    eb = torch.zeros(np_, dtype=torch.int32, device='cuda')
    lv = torch.zeros((S, m, n), dtype=torch.int32, device='cuda')
    Cd = torch.zeros((m, n), dtype=torch.float64, device='cuda')
    _lib.check(
        _lib.lib().sgdml_b200_ozaki_debug(
            m, n, k, Ad.data_ptr(), k, Bd.data_ptr(), k, Cd.data_ptr() if with_product else None, n, S,
            pa.data_ptr(), ea.data_ptr(), pb.data_ptr(), eb.data_ptr(), lv.data_ptr() if with_product else None,
            _lib.current_stream(),
        ),
        'ozaki_debug',
    )
    torch.cuda.synchronize()
    return A, B, pa.cpu().numpy(), ea.cpu().numpy(), pb.cpu().numpy(), eb.cpu().numpy(), lv.cpu().numpy(), Cd.cpu().numpy()


@pytest.mark.parametrize('S', [2, 3, 4, 5, 6, 7])
def test_stage1_split_kernel(S):
    A, B, pa, ea, pb, eb, _, _ = _debug(130, 70, 200, S, with_product=False)
    for X, planes, exps in ((A, pa, ea), (B, pb, eb)):
        e, sl, _ = om.split(X, S)
        rows, k = X.shape
        assert np.array_equal(exps[:rows], e)
        assert np.array_equal(planes[:, :rows, :k].astype(np.float64), sl)
        assert not planes[:, rows:, :].any() and not planes[:, :, k:].any()  # zero padding


@pytest.mark.parametrize('S', [2, 5, 7])
@pytest.mark.parametrize('m,n,k', [(128, 64, 128), (128, 64, 64), (130, 70, 200)])
def test_stage2_raw_level_sums(m, n, k, S):
    A, B, pa, ea, pb, eb, lv, C = _debug(m, n, k, S)
    sa, sb = pa[:, :m, :].astype(np.int64), pb[:, :n, :].astype(np.int64)
    for level in range(2, S + 2):
        want = np.zeros((m, n), dtype=np.int64)
        for p, q in om.level_pairs(S, level):
            want += sa[p - 1] @ sb[q - 1].T
        assert np.array_equal(lv[level - 2].astype(np.int64), want), 'level %d' % level
    assert np.array_equal(C, om.gemm(A, B, np.zeros((m, n)), 1.0, S))


@pytest.mark.parametrize('S,tol_llt,tol_l', [(6, 1e-10, 1e-6), (7, 1e-12, 1e-9)], ids=['6', '7'])
def test_potrf_with_int8_trailing_updates(monkeypatch, S, tol_llt, tol_l):
    """Cholesky with the trailing updates on the int8 path (SGDML_B200_OZAKI_SLICES=6 and 7) against the
    FP64 DMMA factorisation of the same matrix."""
    import torch

    from sgdml_b200 import _lib

    _lib.require_gpu()
    n = 3000
    rng = np.random.default_rng(1)
    G = rng.standard_normal((n, n // 4))
    A = G @ G.T + 1e-3 * np.eye(n)  # condition ~1e6
    outs = {}
    for mode in ('0', str(S)):
        monkeypatch.setenv('SGDML_B200_OZAKI_SLICES', mode)
        Ad = torch.from_numpy(A.copy()).cuda()
        _lib.check(_lib.lib().sgdml_b200_potrf(Ad.data_ptr(), n, n, _lib.current_stream()), 'potrf')
        torch.cuda.synchronize()
        outs[mode] = np.tril(Ad.cpu().numpy())
    L0, LS = outs['0'], outs[str(S)]
    assert rel_err(LS @ LS.T, A) < tol_llt
    assert rel_err(LS, L0) < tol_l


@pytest.mark.parametrize('S', [4, 5, 7], ids=['4', '5', '7'])
def test_large_descriptor_predictor_on_int8_path(monkeypatch, S):
    """GEMM-composed predictor (D > 256) with its four contractions on the int8 path, 4, 5 and 7 slices (set through
    SGDML_B200_OZAKI_PREDICT_SLICES at creation): E and F within the composed bound of the FP64 oracle
    (tests/ozaki_predict_model.py e2e_bound), on the query rows the engine formed."""
    import sgdml_b200
    import ozaki_predict_model as opm
    from sgdml_b200 import synth
    from test_ozaki_predict_classes import tapped

    N, M = 30, 40
    perms = synth.rotor_swap_group(N, 1, 1)
    model = synth.random_model(N, M, perms, 30, seed=2)
    Rq = synth.geometries(N, 9, 1).reshape(9, -1)
    E_ref, F_ref, x, gq, scale, k = opm.oracle_case(model, R=Rq)
    monkeypatch.setenv('SGDML_B200_OZAKI_PREDICT_SLICES', str(S))
    p = sgdml_b200.GDMLPredict(model)
    E, F = p.predict(Rq)
    t, arr, Et, Ft = tapped(p, model, R=Rq)
    assert t['oz_s'] == S
    assert np.array_equal(Et, E) and np.array_equal(Ft, F)
    opm.check_e2e(E, F, E_ref, F_ref, opm.e2e_bound(arr, t['Qg'], t['qq'], gq, S, scale, k), 'S=%d' % S)


@pytest.mark.parametrize('S', [5, 6])
def test_large_descriptor_kmatvec_on_int8_path(monkeypatch, S):
    """K.v of a large-descriptor model (set_alphas refreshes the slices of JA / JA^T; predict_train runs the four
    contractions on the int8 path) against the FP64 DMMA path, 5 slices (the iterative solver's default) and 6."""
    import sgdml_b200
    from sgdml_b200 import synth
    from sgdml_b200.desc import Desc

    N, M = 30, 40
    perms = synth.rotor_swap_group(N, 1, 1)
    model = synth.random_model(N, M, perms, 30, seed=2)
    _, R_d_desc = Desc(N).from_R(synth.geometries(N, M, 2).reshape(M, -1))
    v = np.random.default_rng(3).standard_normal(M * 3 * N)
    out = {}
    for mode in ('0', str(S)):
        monkeypatch.setenv('SGDML_B200_OZAKI_PREDICT_SLICES', mode)
        p = sgdml_b200.GDMLPredict(model)
        p.set_R_d_desc(R_d_desc)
        p.set_alphas(v)
        out[mode] = p.kmatvec_train().copy()
        p.set_alphas(2.0 * v)  # a second set of coefficients through the same handle
        assert rel_err(p.kmatvec_train(), 2.0 * out[mode]) < 1e-9
    assert rel_err(out[str(S)], out['0']) < 1e-8
    # the same through the model-level switch (what the iterative solver uses), back and forth on one handle
    monkeypatch.delenv('SGDML_B200_OZAKI_PREDICT_SLICES')
    p = sgdml_b200.GDMLPredict(model)
    p.set_R_d_desc(R_d_desc)
    p.set_alphas(v)
    kv_fp64 = p.kmatvec_train().copy()
    p.set_contraction_slices(S)
    kv_i8 = p.kmatvec_train().copy()
    p.set_contraction_slices(0)
    assert np.array_equal(p.kmatvec_train(), kv_fp64)
    assert rel_err(kv_i8, out[str(S)]) < 1e-12 and rel_err(kv_fp64, out['0']) < 1e-12
