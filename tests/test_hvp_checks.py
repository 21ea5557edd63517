"""The HVP acceptance checks of tests/hvp_checks.py on CPU: the long-double reference against the torch oracle and
against central differences of its own F near training points; the componentwise bound passed by the NumPy model of
the engine's arithmetic (hvp_oracle.gemm_form_hvp) in every layout class and near training points, and failed by each
injected defect; the chunk plan against hand-computed plans.  No GPU needed."""

import numpy as np
import pytest

import hvp_checks as hc
import hvp_oracle as ho
import predict_checks as pc

FIXTURES = ho.FIXTURES + ['big_c60_m2_s120', 'big_n240_m2_s3']
EPS = (1e-9, 1e-7, 1e-5, 1e-3)


def _v(R, seed):
    return np.random.default_rng(seed).standard_normal(np.shape(R))


def _check(HV, model, R, V, what):
    ratio, tight = hc.check_against_reference(HV, model, R, V, what)
    print('\n[hvp bound] %s: max err/scale %.2e (tau %.2e), tightness %.2e' % (what, ratio, pc.tau(hc.model_terms(model)),
                                                                            tight))
    return ratio, tight


# ------------------------------------------------------------------------------------------------ the reference
def test_reference_refuses_double(monkeypatch):
    """Where long double is only double the reference fails loudly instead of checking FP64 with FP64."""
    model, Rq, _ = ho.fixture_model('n5_m10_s1')
    finfo = np.finfo
    monkeypatch.setattr(np, 'finfo', lambda t: finfo(np.float64))
    with pytest.raises(RuntimeError, match='long'):
        hc.hvp_reference(model, Rq[:1], Rq[:1])


@pytest.mark.parametrize('name', FIXTURES)
def test_reference_matches_torch_oracle(name):
    """At query geometries the long-double reference and the forward-mode torch oracle agree to 1e-12 of the largest
    term (the scale); the torch oracle passes the bound.  pbc_n6_m8 cancels terms ~1e4 times larger than its HV, so
    only the scale-relative agreement is asserted there."""
    model, Rq, _ = ho.fixture_model(name)
    R = Rq[:3]
    V = _v(R, 1)
    F, ref = hc.hvp_reference(model, R, V)
    to = ho.TorchOracle(model)
    HV = to.hvp(R, V)
    scale = hc.hvp_abs_scale(model, R, V)
    ref = ref.astype(np.float64)
    assert np.max(np.abs(HV - ref)) <= 1e-12 * np.max(scale)
    assert np.max(np.abs(to.ef_np(R)[1] - F.astype(np.float64))) <= 1e-12 * np.max(np.abs(F.astype(np.float64))) * (
        100 if name == 'pbc_n6_m8' else 1)
    if name != 'pbc_n6_m8':
        assert np.max(np.abs(HV - ref)) <= 1e-12 * np.max(np.abs(ref))
    _check(HV, model, R, V, '%s torch oracle' % name)


@pytest.mark.parametrize('eps', EPS)
@pytest.mark.parametrize('name', ['n9_m16_s6', 'ecstr_n6_m8', 'pbc_n6_m8', 'big_n100_m2_s12'])
def test_reference_matches_its_central_differences(name, eps):
    """Near training points, where the Matern term (delta.JA)(delta.t)/|delta| has a kink, HV equals central differences
    of the reference's own long-double F, with steps h = min(eps / 10, 1e-6) formed in long double: the kink stays
    outside the stencil, rounding of R + h V does not enter, and F's own rounding (u_ld times the largest term over h)
    stays below 1e-9 of the largest term (the scale)."""
    model, _, Rt = ho.fixture_model(name)
    R = hc.near_training(Rt[:2], eps, 5).astype(hc.LD)
    V = _v(R, 6).astype(hc.LD)
    h = hc.LD(min(eps / 10, 1e-6))
    _, HV = hc.hvp_reference(model, R, V)
    Fp, _ = hc.hvp_reference(model, R + h * V)
    Fm, _ = hc.hvp_reference(model, R - h * V)
    fd = (Fp - Fm) / (2 * h)
    err = np.max(np.abs(HV - fd))
    scale = np.max(hc.hvp_abs_scale(model, R.astype(np.float64), V.astype(np.float64)))
    print('\n[hvp reference] %s eps %g: against central differences %.2e of max |HV|, %.2e of max scale'
          % (name, eps, err / np.max(np.abs(HV)), err / scale))
    assert err <= 1e-9 * scale


# ------------------------------------------------------------------------------------------------ the bound holds
@pytest.mark.parametrize('variant', hc.VARIANTS)
@pytest.mark.parametrize('name', list(hc.CLASSES) + ['big_n240_m2_s3'])
def test_gemm_form_model_passes_in_every_class(name, variant):
    model, _ = hc.class_model(name, variant)
    R, V = hc.queries(model, 3, 11)
    _check(ho.gemm_form_hvp(model, R, V), model, R, V, '%s %s gemm-form model' % (name, variant))


@pytest.mark.parametrize('eps', (0.0,) + EPS)
@pytest.mark.parametrize('name', FIXTURES)
def test_gemm_form_model_passes_near_training_points(name, eps):
    """Exactly on (eps = 0) and near training points the floor under n and the rounding of the expanded x5 stay within
    the bound."""
    model, _, Rt = ho.fixture_model(name)
    R = hc.near_training(Rt[:2], eps, 7)
    V = _v(R, 8)
    _check(ho.gemm_form_hvp(model, R, V), model, R, V, '%s eps %g gemm-form model' % (name, eps))


# ------------------------------------------------------------------------------------------------ the bound bites
def _fails(HV, model, R, V):
    with pytest.raises(AssertionError):
        hc.check_against_reference(HV, model, R, V)


@pytest.mark.parametrize('defect', ['dJ', 'csT', 'pinv_fold'])
@pytest.mark.parametrize('name', ['n9_m16_s6', 'n12_m8_s12', 'big_n100_m2_s12'])
def test_defects_fail(name, defect):
    """A dropped (dJ)^T F_desc term, a dropped (sum c1) T term of dG, a permutation fold through pinv instead of perm."""
    model, Rq, _ = ho.fixture_model(name)
    R = Rq[:3]
    V = _v(R, 9)
    _fails(ho.gemm_form_hvp(model, R, V, defect=defect), model, R, V)


@pytest.mark.parametrize('name', ['ecstr_n6_m8', 'dp112'])
def test_missing_ae_dc2_fails(name):
    if name in hc.CLASSES:
        model, _ = hc.class_model(name, 'ecstr')
        R, V = hc.queries(model, 3, 12)
    else:
        model, Rq, _ = ho.fixture_model(name)
        R, V = Rq[:3], _v(Rq[:3], 12)
    _fails(ho.gemm_form_hvp(model, R, V, defect='ae_dc2'), model, R, V)


@pytest.mark.parametrize('name', ['n9_m16_s6', 'pbc_n6_m8', 'big_c60_m2_s120'])
def test_missing_floor_fails_on_training_points(name):
    model, _, Rt = ho.fixture_model(name)
    R = Rt[:3]
    V = _v(R, 13)
    _fails(ho.gemm_form_hvp(model, R, V, guard=False), model, R, V)


@pytest.mark.parametrize('eps', EPS)
@pytest.mark.parametrize('name', ['n9_m16_s6', 'ecstr_n6_m8', 'big_n100_m2_s12'])
def test_oversized_floor_stays_below_rounding(name, eps):
    """A floor 1e4 times the engine's changes HV by less than the bound at every offset: the floor only replaces dc1 of
    rows within n_floor of the query, and dG sums dc1 (Q - Xc_m) = dc1 delta_m, so its effect on HV is second order in
    |delta| and below the rounding of the expanded sums (sum dc1) Q - sum dc1 Xc_m.  The floor's size is therefore not
    observable; its presence is (test_missing_floor_fails_on_training_points)."""
    model, _, Rt = ho.fixture_model(name)
    R = hc.near_training(Rt[:2], eps, 14)
    V = _v(R, 15)
    _check(ho.gemm_form_hvp(model, R, V, floor_scale=1e4), model, R, V, '%s eps %g floor x 1e4' % (name, eps))


def test_swapped_chunk_edge_rows_fail():
    """One chunk's first row swapped with the previous chunk's last (cap 3: chunks (0, 3), (3, 6), ...)."""
    model, _ = hc.class_model('dp40', 'plain')
    ly = pc.layout(9, 33)
    plan = hc.hvp_chunk_plan(ly, 6, 8, cap=3)
    assert plan.chunks == [(0, 3), (3, 6), (6, 8)] and plan.edges == [0, 2, 3, 5, 6, 7]
    R, V = hc.queries(model, 8, 16)
    HV = ho.gemm_form_hvp(model, R, V)
    hc.check_against_reference(HV, model, R, V)
    HV[[2, 3]] = HV[[3, 2]]
    _fails(HV, model, R, V)


@pytest.mark.parametrize('name', ['n9_m16_s6', 'pbc_n6_m8'])
def test_one_entry_moved_fails(name):
    model, Rq, _ = ho.fixture_model(name)
    R = Rq[:3]
    V = _v(R, 17)
    _, ref = hc.hvp_reference(model, R, V)
    scale = hc.hvp_abs_scale(model, R, V)
    k = hc.model_terms(model)
    HV = ho.gemm_form_hvp(model, R, V)
    i = (1, 5)
    HV[i] += 10 * pc.tau(k) * scale[i]
    with pytest.raises(AssertionError, match='1 HV entries'):
        hc.check_hvp(HV, ref, scale, k)


# ------------------------------------------------------------------------------------------------ chunk plans
def test_chunk_plan_aspirin():
    # a stacked row is 228 + 2 * 1008 + 224 + 2 = 2 470 doubles: 2^31 / (8 * 2 470) = 108 678 rows, 2 * 6 per geometry:
    # 9 056 geometries per chunk
    ly = pc.layout(21, 1000)
    assert hc.hvp_chunk_geos(ly, 6) == 9056
    p = hc.hvp_chunk_plan(ly, 6, 2 * 9056 + 3)
    assert p.chunk == 9056 and p.chunks == [(0, 9056), (9056, 18112), (18112, 18115)]
    assert p.edges == [0, 9055, 9056, 18111, 18112, 18114]
    assert hc.hvp_chunk_plan(ly, 6, 19975, cap=1000).chunks[-1] == (19000, 19975)


def test_chunk_plan_small_models_hit_the_cap():
    # N = 6, S = 2, M = 33: 2^31 / (8 (44 + 2 * 64 + 40 + 2)) = 1 254 371 rows, 313 592 geometries -> 65 536
    ly = pc.layout(6, 33)
    assert (ly.DP, ly.Mpad) == (40, 64)
    p = hc.hvp_chunk_plan(ly, 2, 65536 + 3)
    assert p.chunk == 65536 and p.chunks == [(0, 65536), (65536, 65539)]
    assert p.edges == [0, 65535, 65536, 65538]
    assert hc.hvp_chunk_plan(ly, 2, 0).chunks == []


def test_chunk_plan_large_descriptors():
    # big_n240_m2_s3: DP = 28 680, Mpad = 8: 2^31 / (8 (28 684 + 16 + 28 680 + 2)) = 4 678 rows / (2 * 3) = 779
    ly = pc.layout(240, 2)
    assert (ly.DP, ly.Mpad, ly.large) == (28680, 8, True)
    assert hc.hvp_chunk_geos(ly, 3) == 779
    # ac-ala3-nhme: DP 864, Mpad 2000, S 243: 2^31 / (8 (868 + 4000 + 864 + 2)) = 46 814 rows / (2 * 243) = 96
    assert hc.hvp_chunk_geos(pc.layout(42, 2000), 243) == 96
    assert hc.hvp_chunk_plan(pc.layout(42, 2000), 243, 10, cap=4).chunks == [(0, 4), (4, 8), (8, 10)]
    assert hc.hvp_chunk_geos(pc.layout(42, 2000), 243 * 1000) == 1  # at least one geometry
