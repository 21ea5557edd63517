"""Bring-up harness for the wgmma FP64-via-INT8 GEMM (csrc/ozaki.cu): against NumPy FP64 and against an
exact NumPy model of the slicing.  GPU only."""

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(params=['128', '64'], autouse=True)
def unit_width(request, monkeypatch):
    """Both pipeline-unit widths of the kernel: 128-byte swizzle (9-slot ring) first -- the layout every library
    GEMM uses, so failures there point at the kernel logic rather than at the 64-byte swizzle descriptors."""
    monkeypatch.setenv('SGDML_B200_OZAKI_BK', request.param)
    return request.param


def _run(m, n, k, S, tri=False, alpha=1.0, seed=0, scale_rows=False):
    import torch

    from sgdml_b200 import _lib

    _lib.require_gpu()
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((m, k))
    B = A if tri else rng.standard_normal((n, k))
    if scale_rows:  # rows of very different magnitude: the per-row exponents matter
        A = A * np.exp2(rng.integers(-20, 20, size=(m, 1)).astype(np.float64))
        if not tri:
            B = B * np.exp2(rng.integers(-20, 20, size=(n, 1)).astype(np.float64))
        else:
            B = A
    C0 = rng.standard_normal((m, n))
    Ad = torch.from_numpy(A).cuda()
    Bd = Ad if tri else torch.from_numpy(B).cuda()
    Cd = torch.from_numpy(C0).cuda()
    _lib.check(
        _lib.lib().sgdml_b200_ozaki_gemm_nt(
            m, n, k, float(alpha), Ad.data_ptr(), k, Bd.data_ptr(), k, Cd.data_ptr(), n, S, 1 if tri else 0, _lib.current_stream()
        ),
        'ozaki_gemm_nt',
    )
    torch.cuda.synchronize()
    return A, B, C0, Cd.cpu().numpy()


def _scale(A, B):
    return np.abs(A) @ np.abs(B).T  # componentwise error bound of a dot product


# ------------------------------------------------------------------------------------------------
# Staged bring-up: (1) the split kernel alone, (2) the raw int32 level sums of one tile against exact
# NumPy integer products, (3) everything above.  Run in this order when the kernel first meets hardware:
#   pytest tests/test_ozaki.py -x -q -k "stage1 or stage2"
def _np_split(A, S, bits=7):
    amax = np.max(np.abs(A), axis=1)
    e = np.zeros(len(A), dtype=np.int64)
    nz = amax > 0
    e[nz] = np.frexp(amax[nz])[1] + 1
    r = A / np.exp2(e)[:, None]
    out = np.empty((S,) + A.shape, dtype=np.int64)
    for p in range(S):
        r = r * (1 << bits)
        q = np.rint(r)
        out[p] = q.astype(np.int64)
        r = r - q
    return e, out


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


def test_stage1_split_kernel():
    A, B, pa, ea, pb, eb, _, _ = _debug(130, 70, 200, 7, with_product=False)
    for X, planes, exps in ((A, pa, ea), (B, pb, eb)):
        e, sl = _np_split(X, 7)
        rows, k = X.shape
        assert np.array_equal(exps[:rows], e)
        assert np.array_equal(planes[:, :rows, :k].astype(np.int64), sl)
        assert not planes[:, rows:, :].any() and not planes[:, :, k:].any()  # zero padding


@pytest.mark.parametrize('m,n,k', [(128, 64, 128), (128, 64, 64), (130, 70, 200)])
def test_stage2_raw_level_sums(m, n, k):
    S = 7
    A, B, pa, ea, pb, eb, lv, C = _debug(m, n, k, S)
    sa, sb = pa[:, :m, :].astype(np.int64), pb[:, :n, :].astype(np.int64)
    for level in range(2, S + 2):
        want = np.zeros((m, n), dtype=np.int64)
        for p in range(1, S + 1):
            q = level - p
            if 1 <= q <= S:
                want += sa[p - 1] @ sb[q - 1].T
        assert np.array_equal(lv[level - 2].astype(np.int64), want), 'level %d' % level
    ref = A @ B.T
    assert np.max(np.abs(C - ref) / (np.abs(A) @ np.abs(B).T)) < 1e-12


@pytest.mark.parametrize('m,n,k', [(128, 64, 128), (128, 64, 256), (256, 128, 128), (300, 200, 130), (129, 65, 1000), (64, 8, 40)])
def test_ozaki_gemm_matches_fp64(m, n, k):
    A, B, C0, C = _run(m, n, k, 7)
    ref = C0 + A @ B.T
    assert np.max(np.abs(C - ref) / (_scale(A, B) + 1e-300)) < 1e-12


def test_ozaki_gemm_row_scaling_and_alpha():
    A, B, C0, C = _run(200, 136, 384, 7, alpha=-1.0, scale_rows=True, seed=3)
    ref = C0 - A @ B.T
    assert np.max(np.abs(C - ref) / (_scale(A, B) + np.abs(C0) + 1e-300)) < 1e-12


def test_ozaki_gemm_tri():
    A, B, C0, C = _run(384, 384, 256, 7, tri=True, alpha=-1.0, seed=5)
    ref = C0 - A @ A.T
    il = np.tril_indices(384)
    assert np.max(np.abs(C[il] - ref[il]) / (_scale(A, A)[il] + 1e-300)) < 1e-12


@pytest.mark.parametrize('S', [4, 5, 6, 7])
def test_ozaki_gemm_slice_count(S):
    """The error falls by 2^-7 per slice (tools/ozaki_study.py: 7e-8, 1e-10, 4e-12, 2e-14 for S = 4..7)."""
    A, B, C0, C = _run(256, 192, 512, S, seed=7)
    err = rel_err(C - C0, A @ B.T)
    assert err < 4.0 * 2.0 ** (-7 * S + 4)


def test_potrf_with_int8_trailing_updates(monkeypatch):
    """Cholesky with the trailing updates on the int8 path (SGDML_B200_OZAKI_SLICES=7) against the
    FP64 DMMA factorisation of the same matrix."""
    import torch

    from sgdml_b200 import _lib

    _lib.require_gpu()
    n = 3000
    rng = np.random.default_rng(1)
    G = rng.standard_normal((n, n // 4))
    A = G @ G.T + 1e-3 * np.eye(n)  # condition ~1e6
    outs = {}
    for mode in ('0', '7'):
        monkeypatch.setenv('SGDML_B200_OZAKI_SLICES', mode)
        Ad = torch.from_numpy(A.copy()).cuda()
        _lib.check(_lib.lib().sgdml_b200_potrf(Ad.data_ptr(), n, n, _lib.current_stream()), 'potrf')
        torch.cuda.synchronize()
        outs[mode] = np.tril(Ad.cpu().numpy())
    L0, L7 = outs['0'], outs['7']
    assert rel_err(L7 @ L7.T, A) < 1e-12
    assert rel_err(L7, L0) < 1e-9


def test_large_descriptor_predictor_on_int8_path(monkeypatch):
    """GEMM-composed predictor (D > 256) with its four contractions on the int8 path, 4 and 5
    slices: forces against the oracle (tools/ozaki_study.py predict: 8.8e-9 / 6.5e-11)."""
    import sgdml_b200
    from oracle import predict as opredict
    from sgdml_b200 import synth

    N, M = 30, 40
    perms = synth.rotor_swap_group(N, 1, 1)
    model = synth.random_model(N, M, perms, 30, seed=2)
    Rq = synth.geometries(N, 9, 1).reshape(9, -1)
    E_ref, F_ref = opredict.Predictor(model).predict(Rq)
    for S, tol in ((4, 1e-6), (5, 1e-8), (7, 1e-11)):
        monkeypatch.setenv('SGDML_B200_OZAKI_PREDICT_SLICES', str(S))
        E, F = sgdml_b200.GDMLPredict(model).predict(Rq)
        assert rel_err(F, F_ref) < tol and rel_err(E, E_ref) < tol


def test_large_descriptor_kmatvec_on_int8_path(monkeypatch):
    """K.v of a large-descriptor model (set_alphas refreshes the slices of JA / JA^T; predict_train runs the four
    contractions on the int8 path) against the FP64 DMMA path, 5 slices."""
    import sgdml_b200
    from sgdml_b200 import synth
    from sgdml_b200.desc import Desc

    N, M = 30, 40
    perms = synth.rotor_swap_group(N, 1, 1)
    model = synth.random_model(N, M, perms, 30, seed=2)
    _, R_d_desc = Desc(N).from_R(synth.geometries(N, M, 2).reshape(M, -1))
    v = np.random.default_rng(3).standard_normal(M * 3 * N)
    out = {}
    for S in ('0', '5'):
        monkeypatch.setenv('SGDML_B200_OZAKI_PREDICT_SLICES', S)
        p = sgdml_b200.GDMLPredict(model)
        p.set_R_d_desc(R_d_desc)
        p.set_alphas(v)
        out[S] = p.kmatvec_train().copy()
        p.set_alphas(2.0 * v)  # a second set of coefficients through the same handle
        assert rel_err(p.kmatvec_train(), 2.0 * out[S]) < 1e-9
    assert rel_err(out['5'], out['0']) < 1e-8
    # the same through the model-level switch (what the iterative solver uses), back and forth on one handle
    monkeypatch.delenv('SGDML_B200_OZAKI_PREDICT_SLICES')
    p = sgdml_b200.GDMLPredict(model)
    p.set_R_d_desc(R_d_desc)
    p.set_alphas(v)
    kv_fp64 = p.kmatvec_train().copy()
    p.set_contraction_slices(5)
    kv_i8 = p.kmatvec_train().copy()
    p.set_contraction_slices(0)
    assert np.array_equal(p.kmatvec_train(), kv_fp64)
    assert rel_err(kv_i8, out['5']) < 1e-12 and rel_err(kv_fp64, out['0']) < 1e-12
