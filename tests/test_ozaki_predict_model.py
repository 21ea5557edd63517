"""The stage model of the large-descriptor predictor (tests/ozaki_predict_model.py) on the CPU: the int8-slice
composition it states stays within the composed bound of the FP64 oracle at every slice count, model kind and at
training points; the bound is not vacuous; and every fault the device checks are meant to catch fails its check."""

import numpy as np
import pytest

import ozaki_predict_model as opm

N, M = 24, 29  # D = 276 > 256: the GEMM-composed path; Mpad = 32 leaves three padding columns


@pytest.fixture(scope='module')
def cases():
    """Per model kind: (model, arrays, query case, training-point case); a case is (xq, gq, E_ref, F_ref, scale, k)."""
    out = {}
    for i, kind in enumerate(opm.KINDS):
        model, R, g = opm.make_model(N, M, kind, seed=3 + i)
        arr = opm.layout_arrays(model)
        Rq = opm.queries(model, 3, seed=40 + i)
        E, F, x, gq, scale, k = opm.oracle_case(model, R=Rq)
        rows = np.array([0, 7, M - 1])
        Et, Ft, xt, gt, st, kt = opm.oracle_case(model, train=(arr['X'][rows], g[rows]))
        out[kind] = (model, arr, (x, gq, E, F, scale, k), (xt, gt, Et, Ft, st, kt))
    return out


def _run(arr, case, S, **kw):
    x, gq = case[0], case[1]
    Qg, qq = opm.query_rows(x, arr['pinv'], arr['mu'], arr['DS'])
    t = opm.stages(arr, Qg, qq, S, **kw)
    E, F, _ = opm.finish(t['G'], t['Erow'], arr['perm'], gq, arr['std'], arr['c'])
    return Qg, qq, t, E, F


@pytest.mark.parametrize('S', [0, 2, 3, 4, 5, 6, 7])
@pytest.mark.parametrize('kind', opm.KINDS)
@pytest.mark.parametrize('where', ['queries', 'train'])
def test_slice_model_within_composed_bound(cases, kind, S, where):
    model, arr, qcase, tcase = cases[kind]
    case = qcase if where == 'queries' else tcase
    x, gq, E_ref, F_ref, scale, k = case
    Qg, qq, t, E, F = _run(arr, case, S)
    opm.check_query_rows(t, arr, x)
    opm.check_stages(t, arr, S, gq=gq, E=E, F=F)
    bound = opm.e2e_bound(arr, Qg, qq, gq, S, scale, k)
    opm.check_e2e(E, F, E_ref, F_ref, bound, '%s %s S=%d' % (kind, where, S))


# the int8 part of the force bound is within this factor of the worst entry's actual int8 error (observed: 14 to 70)
BOUND_FACTOR = 100.0


@pytest.mark.parametrize('S', [2, 3, 4, 5, 6, 7])
def test_composed_bound_is_not_vacuous(cases, S):
    """The int8 part of the bound against the int8 error itself (the slice model against its own FP64 chain): the
    worst force entry reaches at least 1/BOUND_FACTOR of its bound."""
    for kind in ('plain', 'perms'):
        _, arr, case, _ = cases[kind]
        Qg, qq, t, E, F = _run(arr, case, S)
        _, _, _, E0, F0 = _run(arr, case, 0)
        _, _, (dE, dF) = opm.e2e_bound(arr, Qg, qq, case[1], S, case[4], case[5])
        ratio = np.max(np.abs(F - F0) / dF)
        assert ratio <= 1.0, (kind, S, ratio)
        assert ratio >= 1.0 / BOUND_FACTOR, (kind, S, ratio)


def _defect_case(cases, defect):
    kind = 'ecstr' if defect == 'drop_ae' else 'perms'
    model, arr, case, tcase = cases[kind]
    prev = None
    if defect == 'stale_ja':
        prev = dict(arr, JA=arr['JA'] * 0.5, JAT=arr['JAT'] * 0.5)  # the coefficients before set_alphas(2 v)
    elif defect == 'foreign_xc':
        prev = opm.layout_arrays(cases['plain'][0])
    elif defect == 'stale_row':
        prev = opm.query_rows(tcase[0][:1], arr['pinv'], arr['mu'], arr['DS'])[0]
    return arr, case, prev


@pytest.mark.parametrize('S', [2, 5, 7])
@pytest.mark.parametrize('defect', opm.DEFECTS)
def test_defect_fails_its_check(cases, defect, S):
    arr, case, prev = _defect_case(cases, defect)
    _, _, t, E, F = _run(arr, case, S, defect=defect, prev=prev)
    with pytest.raises(AssertionError):
        opm.check_query_rows(t, arr, case[0])
        opm.check_stages(t, arr, S, gq=case[1], E=E, F=F)
