"""Hessian-vector products (sgdml_b200_predict_hvp) in every layout class against the long-double reference of
tests/hvp_checks.py, with its componentwise bound.

Models: one per padded descriptor width of the fused predictor (DP = 40, 72, 112, 160, 224, 256: the DP / DS strides
of the transposed copies XcT / JAT the HVP builds lazily), N = 24 just past 256 (GEMM form), N = 30 and the golden
big_n240_m2_s3; S = 6 (rotor-swap group) except the fixture's 3; M one more than a multiple of BM, so padded training
columns must contribute nothing.  Each runs plain, with random alphas_E and in a skewed cell.  Near training points
(eps = 0 .. 1e-3 A) the floor under n and the rounding of the expanded x5 are exercised; chunk edges at a full
65 536-geometry chunk (k_fdesc_gather's grid-stride loop over y) and at several default-size aspirin chunks; and the
state changes an HVP depends on: set_alphas (refreshing XcT / JAT), set_lattice, the int8-slice setting (which the HVP
ignores: it is always FP64) and an empty batch.  Each check prints the worst |err| / scale against tau and the bound's
tightness, max(tau scale) / max |HV_ref|."""

import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import hvp_checks as hc  # noqa: E402
import predict_checks as pc  # noqa: E402
from oracle import desc as odesc  # noqa: E402

NAMES = list(hc.CLASSES) + ['big_n240_m2_s3']
FUSED = [n for n in hc.CLASSES if not pc.layout(*hc.CLASSES[n]).large]
EPS = (0.0, 1e-9, 1e-7, 1e-5, 1e-3)
NEAR = [('dp112', 'plain'), ('dp224', 'ecstr'), ('dp160', 'pbc'), ('n24', 'plain')]
_REPORT = {}


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


def _check(HV, model, R, V, what, lat_and_inv='model'):
    HV = HV.cpu().numpy() if hasattr(HV, 'cpu') else HV
    ratio, tight = hc.check_against_reference(HV, model, R, V, what, lat_and_inv)
    _REPORT[what] = (ratio, tight)
    print('\n[hvp] %s: max err/scale %.2e (tau %.2e), tightness %.2e'
          % (what, ratio, pc.tau(hc.model_terms(model)), tight))
    return ratio, tight


def _layout(model):
    N = int(np.asarray(model['z']).shape[0])
    return pc.layout(N, int(np.asarray(model['R_desc']).shape[1]))


# ------------------------------------------------------------------------------------------------ classes
@pytest.mark.parametrize('variant', hc.VARIANTS)
@pytest.mark.parametrize('name', NAMES)
def test_hvp_in_every_class(eng, name, variant):
    model, _ = hc.class_model(name, variant)
    ly = _layout(model)
    if name in hc.CLASSES:
        assert ly.Mpad > int(model['R_desc'].shape[1])
        assert ly.large == (name not in FUSED)
    R, V = hc.queries(model, 6 if name == 'big_n240_m2_s3' else 16, 21)
    _check(eng.GDMLPredict(model).predict_hvp(R, V), model, R, V, '%s %s (DP %d)' % (name, variant, ly.DP))


@pytest.mark.parametrize('eps', EPS)
@pytest.mark.parametrize('name,variant', NEAR)
def test_hvp_near_training_points(eng, name, variant, eps):
    model, R_train = hc.class_model(name, variant)
    R = hc.near_training(R_train, eps, 22)
    if 'lattice' in model:
        lat = np.asarray(model['lattice'])
        R = R[pc.pbc_margin(R, lat, np.linalg.inv(lat)) >= hc.PBC_MARGIN]
    R = np.ascontiguousarray(R[:6])
    assert R.shape[0] >= 3
    V = np.random.default_rng(23).standard_normal(R.shape)
    HV = eng.GDMLPredict(model).predict_hvp(R, V)
    assert np.all(np.isfinite(HV))
    _check(HV, model, R, V, '%s %s eps %g' % (name, variant, eps))


# ------------------------------------------------------------------------------------------------ chunk edges
def _edge_rows(plan, width=64):
    rows = set()
    for lo, hi in plan.chunks:
        rows.update(range(lo, min(lo + width, hi)))
        rows.update(range(max(hi - width, lo), hi))
    return sorted(rows)


def test_hvp_full_capped_chunk_and_tail(eng):
    """N = 6, S = 2, M = 33 (Mpad 64): the chunk rule gives 313 592 geometries, capped at 65 536, so B = 65 539 runs one
    full chunk -- k_fdesc_gather's grid stops at y = 65 535 and its grid-stride loop must reach geometry 65 535 -- and a
    tail of 3.  Every row of the first and last 64 geometries of each chunk is checked, and the whole output is
    bit-identical to chunks of 1 000."""
    from sgdml_b200 import synth

    N, M, B = 6, 33, 65536 + 3
    perms = synth.rotor_swap_group(N, 0, 1)
    rng = np.random.default_rng(31)
    model = hc.build_model(synth.geometries(N, M, 31).reshape(M, -1), rng.standard_normal(M * 3 * N), perms)
    plan = hc.hvp_chunk_plan(_layout(model), perms.shape[0], B)
    assert plan.chunks == [(0, 65536), (65536, B)]
    R = synth.geometries(N, B, 32).reshape(B, -1)
    V = rng.standard_normal(R.shape)
    HV = eng.GDMLPredict(model).predict_hvp(R, V)
    rows = _edge_rows(plan)
    assert 65535 in rows and len(rows) == 131
    _check(HV[rows], model, R[rows], V[rows], 'N 6 B %d chunk edges' % B)
    with _chunk_cap(1000):
        HV1 = eng.GDMLPredict(model).predict_hvp(R, V)
    assert np.array_equal(HV, HV1)


def test_hvp_aspirin_default_chunks(eng):
    """The benchmarked aspirin shape (N 21, M 1000, S 6, random coefficients): 9 056 geometries per default (~2 GB)
    chunk, B = 2 chunks + 3, from CUDA tensors.  Chunk-edge rows and a seeded sample of 64 rows against the reference;
    the whole output bit-identical to chunks of 1 000."""
    import torch

    from sgdml_b200 import synth

    cfg = synth.CONFIGS['aspirin']
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, _ = synth.config_perms_and_r0('aspirin')
    model = synth.random_model(N, M, perms, cfg['sig'])
    plan = hc.hvp_chunk_plan(_layout(model), perms.shape[0], 2 * 9056 + 3)
    assert plan.chunk == 9056 and len(plan.chunks) == 3
    B = plan.chunks[-1][1]
    R = synth.geometries(N, B, 41).reshape(B, -1)
    V = np.random.default_rng(42).standard_normal(R.shape)
    Rd, Vd = torch.from_numpy(R).cuda(), torch.from_numpy(V).cuda()
    HV = eng.GDMLPredict(model).predict_hvp(Rd, Vd)
    torch.cuda.synchronize()
    HV = HV.cpu().numpy()
    rows = sorted(set(plan.edges) | set(np.random.default_rng(43).choice(B, 64, replace=False).tolist()))
    _check(HV[rows], model, R[rows], V[rows], 'aspirin B %d edges + sample' % B)
    with _chunk_cap(1000):
        HV1 = eng.GDMLPredict(model).predict_hvp(Rd, Vd)
        torch.cuda.synchronize()
    assert np.array_equal(HV, HV1.cpu().numpy())


# ------------------------------------------------------------------------------------------------ state changes
@pytest.mark.parametrize('name', FUSED)
def test_hvp_after_set_alphas(eng, name):
    """An HVP builds XcT / JAT at the class's DP / DS strides; set_alphas (with alphas_E) must refresh them: the second
    HVP matches the reference of the new coefficients, which move HV by far more than the bound."""
    model, R_train = hc.class_model(name, 'plain')
    M = R_train.shape[0]
    _, g = odesc.from_R(R_train)
    p = eng.GDMLPredict(model)
    p.set_R_d_desc(g)
    R, V = hc.queries(model, 8, 51)
    _check(p.predict_hvp(R, V), model, R, V, '%s before set_alphas' % name)
    rng = np.random.default_rng(52)
    aF, aE = rng.standard_normal(M * R_train.shape[1]), 3.0 * rng.standard_normal(M)
    p.set_alphas(aF, alphas_E=aE)
    model2 = hc.build_model(R_train, aF, model['perms'], model['sig'], alphas_E=aE)
    model2['std'], model2['c'] = model['std'], model['c']
    HV = p.predict_hvp(R, V)
    _, old = hc.hvp_reference(model, R, V)
    _, new = hc.hvp_reference(model2, R, V)
    assert np.max(np.abs(new - old)) > 0.1 * np.max(np.abs(new))
    _check(HV, model2, R, V, '%s after set_alphas' % name)


def test_hvp_after_set_lattice(eng):
    from sgdml_b200 import _lib

    model, _ = hc.class_model('dp72', 'pbc')
    lat2 = np.ascontiguousarray(1.07 * np.asarray(model['lattice']))
    inv2 = np.ascontiguousarray(np.linalg.inv(lat2))
    R, V = hc.queries(model, 24, 61)
    keep = pc.pbc_margin(R, lat2, inv2) >= hc.PBC_MARGIN
    R, V = np.ascontiguousarray(R[keep][:16]), np.ascontiguousarray(V[keep][:16])
    p = eng.GDMLPredict(model)
    HV1 = p.predict_hvp(R, V)
    _check(HV1, model, R, V, 'dp72 model cell')
    _lib.check(_lib.lib().sgdml_b200_model_set_lattice(p._handle, _lib.ptr(lat2), _lib.ptr(inv2)), 'set_lattice')
    HV2 = p.predict_hvp(R, V)
    assert not np.array_equal(HV1, HV2)
    _check(HV2, model, R, V, 'dp72 after set_lattice', lat_and_inv=(lat2, inv2))


def test_hvp_ignores_contraction_slices(eng):
    """The int8-slice setting of large descriptors changes predict, never the HVP: it is always FP64."""
    model, _ = hc.class_model('n30', 'ecstr')
    R, V = hc.queries(model, 8, 71)
    p = eng.GDMLPredict(model)
    HV0 = p.predict_hvp(R, V)
    p.set_contraction_slices(5)
    HV1 = p.predict_hvp(R, V)
    p.set_contraction_slices(0)
    assert np.array_equal(HV0, HV1)
    _check(HV1, model, R, V, 'n30 ecstr with 5 int8 slices set')


def test_hvp_empty_batch(eng):
    model, _ = hc.class_model('dp40', 'plain')
    R = np.empty((0, 27))
    HV = eng.GDMLPredict(model).predict_hvp(R, R.copy())
    assert isinstance(HV, np.ndarray) and HV.shape == (0, 27)


def test_report():
    """Summary of every check above: worst err/scale and tightness per case (run with -s)."""
    if not _REPORT:
        pytest.skip('no HVP checks ran')
    print('\n[hvp report] %-40s %12s %12s' % ('case', 'err/scale', 'tightness'))
    for what, (ratio, tight) in _REPORT.items():
        print('[hvp report] %-40s %12.2e %12.2e' % (what, ratio, tight))
