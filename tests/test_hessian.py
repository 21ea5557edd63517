"""Batched energy Hessians (sgdml_b200_predict_hessian, GDMLPredict.predict_hessian): every column equals
-predict_hvp(R, e_i) bit for bit on golden fixtures and on models of both descriptor classes (plain, alphas_E, periodic),
sampled columns pass the HVP's componentwise bound against the long-double reference, direction blocks and chunks do
not change a bit, host / device / pinned buffers, B = 0, rejected calls, one 370-atom geometry, and HVP and Hessian
calls interleaved on one workspace."""

import numpy as np
import pytest

import hvp_checks as hc
import hvp_oracle

pytestmark = pytest.mark.gpu


def _gp(model):
    import sgdml_b200

    return sgdml_b200.GDMLPredict(model)


def _columns_by_hvp(gp, R, cols=None):
    """H[b][:, i] = -predict_hvp(R[b], e_i) for the columns `cols` (all by default): (B, 3N, len(cols))."""
    B, n = R.shape
    cols = range(n) if cols is None else cols
    out = np.empty((B, n, len(cols)))
    for j, i in enumerate(cols):
        V = np.zeros_like(R)
        V[:, i] = 1.0
        out[:, :, j] = -gp.predict_hvp(R, V)
    return out


def _chunk(n):
    from sgdml_b200 import _lib

    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(int(n)), 'set_predict_chunk')


@pytest.mark.parametrize('name', ['n9_m16_s6', 'n21_m6_s6', 'ecstr_n6_m8', 'pbc_n6_m8'])
def test_columns_are_the_hvp_bit_for_bit_golden(name):
    model, Rq, _ = hvp_oracle.fixture_model(name)
    gp = _gp(model)
    R = np.ascontiguousarray(Rq[:5])
    H = gp.predict_hessian(R)
    assert H.shape == (len(R), R.shape[1], R.shape[1])
    assert np.array_equal(H, _columns_by_hvp(gp, R))
    print('%s: max |H - H^T| / max |H| = %.2e' % (name, np.max(np.abs(H - H.transpose(0, 2, 1))) / np.max(np.abs(H))))


@pytest.mark.parametrize('name, variant', [('dp40', 'plain'), ('dp72', 'ecstr'), ('dp224', 'pbc'), ('n24', 'plain'),
                                           ('n24', 'ecstr'), ('n30', 'pbc')])
def test_columns_are_the_hvp_bit_for_bit_classes(name, variant):
    """Both descriptor classes (D <= 256: the fused predictor's models; D > 256: the GEMM-composed form), with alphas_E
    and in a cell; sampled columns also against the long-double reference."""
    model, _ = hc.class_model(name, variant)
    gp = _gp(model)
    R, _ = hc.queries(model, 3, seed=11)
    H = gp.predict_hessian(R)
    assert np.array_equal(H, _columns_by_hvp(gp, R))
    n = R.shape[1]
    for i in (0, n // 2, n - 1):
        V = np.zeros_like(R)
        V[:, i] = 1.0
        hc.check_against_reference(-H[:, :, i], model, R, V, what='%s/%s col %d' % (name, variant, i))


@pytest.mark.parametrize('name', ['n9_m16_s6', 'n24'])
def test_direction_blocks_and_chunks_are_bit_identical(name):
    """Caps of 1 (one direction per block), 4 (blocks of 7 directions, a geometry split over several) and 200 (whole
    geometries, several per chunk, several chunks) against the uncapped call."""
    if name == 'n24':
        model, _ = hc.class_model(name, 'ecstr')
        R, _ = hc.queries(model, 7, seed=5)
    else:
        model, Rq, _ = hvp_oracle.fixture_model(name)
        R = np.ascontiguousarray(Rq[:7])
    gp = _gp(model)
    ref = gp.predict_hessian(R)
    try:
        for cap in (1, 4, 200):
            _chunk(cap)
            assert np.array_equal(gp.predict_hessian(R), ref), cap
    finally:
        _chunk(0)


def test_buffers_empty_batch_and_rejected_calls():
    import torch

    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model('n9_m16_s6')
    gp = _gp(model)
    R = np.ascontiguousarray(Rq[:4])
    n = R.shape[1]
    ref = gp.predict_hessian(R)
    Rt = torch.from_numpy(R).cuda()
    Hd = gp.predict_hessian(Rt)
    assert Hd.is_cuda and np.array_equal(Hd.cpu().numpy(), ref)
    Hp = gp.predict_hessian(torch.from_numpy(R).pin_memory())
    assert Hp.is_pinned() and np.array_equal(Hp.numpy(), ref)
    out = np.full((4, n, n), 7.0)
    assert gp.predict_hessian(R, out=out) is out and np.array_equal(out, ref)
    assert np.array_equal(gp.predict_hessian(R[1]), ref[1:2])  # one geometry without its batch axis
    assert gp.predict_hessian(np.empty((0, n))).shape == (0, n, n)
    with pytest.raises(ValueError):
        gp.predict_hessian(R, out=np.empty((4, n, n - 1)))
    with pytest.raises(ValueError):
        gp.predict_hessian(Rt, out=np.empty((4, n, n)))  # host buffer for a CUDA input
    L = _lib.lib()
    H = np.full((4, n, n), 7.0)
    s = _lib.current_stream()
    assert L.sgdml_b200_predict_hessian(None, R.ctypes.data, 4, H.ctypes.data, s) <= -1000
    assert L.sgdml_b200_predict_hessian(gp._handle, None, 4, H.ctypes.data, s) <= -1000
    assert L.sgdml_b200_predict_hessian(gp._handle, R.ctypes.data, 4, None, s) <= -1000
    assert L.sgdml_b200_predict_hessian(gp._handle, R.ctypes.data, -1, H.ctypes.data, s) <= -1000
    assert np.all(H == 7.0)
    assert L.sgdml_b200_predict_hessian(gp._handle, R.ctypes.data, 0, H.ctypes.data, s) == 0
    assert np.all(H == 7.0)


def test_370_atoms():
    """H is 1110 x 1110; sampled columns bit for bit against the HVP."""
    model, Rq, _ = hvp_oracle.fixture_model('big_n370_m2_s3')
    gp = _gp(model)
    R = np.ascontiguousarray(Rq[:1])
    H = gp.predict_hessian(R)
    assert H.shape == (1, 1110, 1110) and np.all(np.isfinite(H))
    cols = [0, 1, 554, 1108, 1109]
    assert np.array_equal(H[:, :, cols], _columns_by_hvp(gp, R, cols))


def test_hvp_and_hessian_share_one_workspace():
    """predict_hvp and predict_hessian share one workspace that grows to the largest request and never shrinks: calls
    interleaved on one model, with growing and shrinking batches, host and device buffers and a chunk cap set and cleared
    in between, each bit-identical to the same call on a fresh model."""
    import torch

    model, _ = hc.class_model('n24', 'ecstr')
    R, V = hc.queries(model, 40, seed=9)

    def call(gp, kind, B, dev):
        Rb, Vb = R[:B], V[:B]
        if dev:
            Rb, Vb = torch.from_numpy(Rb).cuda(), torch.from_numpy(Vb).cuda()
        out = gp.predict_hessian(Rb) if kind == 'hessian' else gp.predict_hvp(Rb, Vb)
        return out.cpu().numpy() if dev else out

    gp = _gp(model)
    calls = [('hessian', 3, False, 0), ('hvp', 40, False, 0), ('hessian', 7, True, 0), ('hvp', 2, True, 0),
             ('hessian', 2, False, 4), ('hvp', 40, True, 4), ('hessian', 1, True, 1), ('hvp', 9, False, 0),
             ('hessian', 7, False, 0), ('hvp', 1, False, 1), ('hessian', 5, True, 0), ('hvp', 40, False, 0)]
    try:
        for kind, B, dev, cap in calls:
            _chunk(cap)
            assert np.array_equal(call(gp, kind, B, dev), call(_gp(model), kind, B, dev)), (kind, B, dev, cap)
    finally:
        _chunk(0)
