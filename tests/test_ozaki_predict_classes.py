"""The large-descriptor predictor (D > 256) on the device, stage by stage, against the stage model
tests/ozaki_predict_model.py: every int8 contraction bit for bit against tests/ozaki_model.py on the operands the kernel
was fed (sgdml_b200_predict_stages), the FP64 stages within their tolerances, E and F within the composed bound of the
FP64 oracle at every slice count, every call path bit-identical to the tapped rows, and every model-state transition
bit-identical to a fresh model in the same state.  GPU only."""

import ctypes

import numpy as np
import pytest

import ozaki_model as om
import ozaki_predict_model as opm
import predict_checks as pc

pytestmark = pytest.mark.gpu

SLICES = (0, 2, 3, 4, 5, 6, 7)
DOCUMENTED = {4: 8.8e-9, 5: 6.5e-11, 6: 5.4e-13}  # the NumPy study's figures (tools/ozaki_study.py predict, N = 21)
_ARRAYS = ('Qg', 'qq', 'S1', 'S2', 'C1', 'C2', 'csum', 'Erow', 'acc', 'G', 'Xc', 'JA', 'XcT', 'JAT', 'mm', 'xja', 'mu',
           'ae')


class _Taps(ctypes.Structure):
    _fields_ = [(n, ctypes.c_void_p) for n in _ARRAYS] + [
        ('oz_s', ctypes.c_int), ('use_ae', ctypes.c_int), ('DS', ctypes.c_int64), ('DP', ctypes.c_int64),
        ('Mpad', ctypes.c_int64)]


@pytest.fixture(autouse=True)
def _clean_env(monkeypatch):
    monkeypatch.delenv('SGDML_B200_OZAKI_PREDICT_SLICES', raising=False)
    monkeypatch.delenv('SGDML_B200_OZAKI_DBG', raising=False)


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    yield sgdml_b200
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(0), 'set_predict_chunk')


def _device_levels(sa, sb, S):
    """om.levels with the products on the device (exact: integer operands, partial sums far below 2^53)."""
    import torch

    ta = torch.from_numpy(np.ascontiguousarray(sa)).cuda()
    tb = torch.from_numpy(np.ascontiguousarray(sb)).cuda()
    out = []
    for L in range(2, S + 2):
        acc = None
        for p, q in om.level_pairs(S, L):
            t = ta[p - 1] @ tb[q - 1].T
            acc = t if acc is None else acc + t
        out.append(acc.cpu().numpy())
    return out


def tapped(p, model, R=None, n_geo=None, m_begin=0, scaled=1, stages=True):
    """One chunk through sgdml_b200_predict_stages: (taps dict, arrays dict of the model at call time, E, F).  R: host
    array of queries (copied to the device) or None for training points m_begin .. m_begin + n_geo - 1."""
    import torch

    from sgdml_b200 import _lib

    N = int(np.asarray(model['z']).shape[0])
    M = int(model['R_desc'].shape[1])
    S_p = int(np.asarray(model['perms']).shape[0])
    ly = pc.layout(N, M)
    DS, DP, Mpad = ly.DP + 4, ly.DP, ly.Mpad
    n = R.shape[0] if R is not None else n_geo
    rows = n * S_p
    shapes = dict(Qg=(rows, DS), qq=(rows,), S1=(rows, Mpad), S2=(rows, Mpad), C1=(rows, Mpad), C2=(rows, Mpad),
                  csum=(rows,), Erow=(rows,), acc=(rows, DP), G=(rows, DP), Xc=(Mpad, DS), JA=(Mpad, DS),
                  XcT=(DP, Mpad), JAT=(DP, Mpad), mm=(Mpad,), xja=(Mpad,), mu=(DS,), ae=(Mpad,))
    bufs = {k: torch.full(v, np.nan, dtype=torch.float64, device='cuda') for k, v in shapes.items()} if stages else {}
    taps = _Taps(**{k: b.data_ptr() for k, b in bufs.items()})
    E = torch.empty(n, dtype=torch.float64, device='cuda')
    F = torch.empty((n, 3 * N), dtype=torch.float64, device='cuda')
    Rd = torch.from_numpy(np.ascontiguousarray(R)).cuda() if R is not None else None
    _lib.check(
        _lib.lib().sgdml_b200_predict_stages(p._handle, None if Rd is None else Rd.data_ptr(), n, m_begin, scaled,
                                             ctypes.addressof(taps), E.data_ptr(), F.data_ptr(),
                                             _lib.current_stream()),
        'predict_stages')
    assert (taps.DS, taps.DP, taps.Mpad) == (DS, DP, Mpad)
    t = {k: b.cpu().numpy() for k, b in bufs.items()}
    t['oz_s'] = taps.oz_s
    arr = opm.layout_arrays(model)
    if stages:
        for k in ('Xc', 'JA', 'XcT', 'JAT', 'mm', 'xja', 'mu', 'ae'):
            arr[k] = t[k]
        arr['use_ae'] = bool(taps.use_ae)
    return t, arr, E.cpu().numpy(), F.cpu().numpy()


def _predictor(eng, model, S, R_d_desc=None):
    p = eng.GDMLPredict(model)
    if S:
        p.set_contraction_slices(S)
    if R_d_desc is not None:
        p.set_R_d_desc(R_d_desc)
    return p


def _same(what, got, want):
    opm.check_exact(what, np.asarray(got), np.asarray(want))


_CASES = {}


def _case(kind, N=24, M=29, B=3, seed=0, perms=None, r0=None):
    """(model, R_train, g_train, Rq, oracle query case, oracle training case on rows 5..7) per kind and shape, cached."""
    key = (kind, N, M, B, seed)
    if key not in _CASES:
        model, R, g = opm.make_model(N, M, kind, seed=seed, perms=perms, r0=r0)
        Rq = opm.queries(model, B, seed=50 + seed)
        q = opm.oracle_case(model, R=Rq)
        rows = np.arange(5, 8)
        X = np.asarray(model['R_desc']).T
        tc = opm.oracle_case(model, train=(X[rows], g[rows]))
        _CASES[key] = (model, R, g, Rq, q, tc)
    return _CASES[key]


# ------------------------------------------------------------------------------------------------ a. + b.
_REPORT = {}


@pytest.mark.parametrize('S', SLICES)
@pytest.mark.parametrize('kind', opm.KINDS)
def test_stages_and_end_to_end(eng, kind, S):
    """N = 24, M = 29 (DS = 284, Mpad = 32: padding columns): random queries and training points 5..7 (R = NULL, the
    self-pair at n = 0), every stage against the stage model, E and F within the composed bound."""
    model, R, g, Rq, (E_ref, F_ref, x, gq, scale, k), tcase = _case(kind)
    p = _predictor(eng, model, S, R_d_desc=g)
    t, arr, E, F = tapped(p, model, R=Rq)
    assert t['oz_s'] == S
    opm.check_stages(t, arr, S)
    Qg, qq = t['Qg'], t['qq']
    rF, _ = opm.check_e2e(E, F, E_ref, F_ref, opm.e2e_bound(arr, Qg, qq, gq, S, scale, k), '%s S=%d' % (kind, S))
    rel = float(np.max(np.abs(F - F_ref)) / np.max(np.abs(F_ref)))
    # training points: Qg bit for bit from the training descriptors, the finishing from the cached Jacobians
    Et_ref, Ft_ref, xt, gt, st, kt = tcase
    t2, arr2, E2, F2 = tapped(p, model, n_geo=3, m_begin=5, scaled=1)
    opm.check_query_rows(t2, arr2, xt)
    opm.check_stages(t2, arr2, S, gq=gt, E=E2, F=F2)
    opm.check_e2e(E2, F2, Et_ref, Ft_ref, opm.e2e_bound(arr2, t2['Qg'], t2['qq'], gt, S, st, kt), 'train S=%d' % S)
    rel = max(rel, float(np.max(np.abs(F2 - Ft_ref)) / np.max(np.abs(Ft_ref))))
    _REPORT[(kind, S)] = rel
    print('\n%s S=%d: forces max rel err vs FP64 oracle %.2e (documented %s), worst |dF| / bound %.2e'
          % (kind, S, rel, DOCUMENTED.get(S, '-'), rF))


@pytest.mark.parametrize('name', ['ac-ala3-nhme', 'c60'])
def test_stages_large_symmetry_groups(eng, name):
    """The permutation-heavy shapes at the solver's 5 slices: Ac-Ala3-NHMe (N = 42, 243 permutations; M = 200 here)
    and C60 (N = 60, 120 permutations; M = 40): contractions bit for bit (levels on the device), stages, bound."""
    from sgdml_b200 import synth

    perms, r0 = synth.config_perms_and_r0(name)
    N = perms.shape[1]
    M = 200 if name == 'ac-ala3-nhme' else 40
    model, R, g, Rq, (E_ref, F_ref, x, gq, scale, k), _ = _case('perms', N=N, M=M, B=1, seed=7, perms=perms, r0=r0)
    p = _predictor(eng, model, 5)
    t, arr, E, F = tapped(p, model, R=Rq)
    assert t['oz_s'] == 5
    opm.check_stages(t, arr, 5, product=_device_levels)
    opm.check_e2e(E, F, E_ref, F_ref, opm.e2e_bound(arr, t['Qg'], t['qq'], gq, 5, scale, k), name)


def test_largest_int8_shape(eng):
    """N = 181 (DS = 16300, the largest descriptor the int8 path takes): stages bit for bit at 7 slices; N = 182 falls
    back to FP64 (slices 0) and is bit-identical to a model set to 0."""
    for N, want in ((181, 7), (182, 0)):
        model, _, g = opm.make_model(N, 9, 'plain', seed=1)
        Rq = opm.queries(model, 2, seed=3)
        p = _predictor(eng, model, 7)
        t, arr, E, F = tapped(p, model, R=Rq, stages=(N == 181))
        assert t['oz_s'] == want
        if N == 181:
            opm.check_stages(t, arr, 7, product=_device_levels)
        else:
            E0, F0 = _predictor(eng, model, 0).predict(Rq)
            _same('N = 182 at 7 slices vs 0: F', F, F0)
            _same('N = 182 at 7 slices vs 0: E', E, E0)


def test_training_count_limit(eng):
    """Mpad <= 16384 takes slices: M = 16384 reports 5, M = 16385 reports 0 and is bit-identical to FP64."""
    for M, want in ((16384, 5), (16385, 0)):
        model, _, _ = opm.make_model(24, M, 'plain', seed=2)
        Rq = opm.queries(model, 1, seed=4)
        p = _predictor(eng, model, 5)
        t, _, E, F = tapped(p, model, R=Rq, stages=False)
        assert t['oz_s'] == want
        if want == 0:
            E0, F0 = _predictor(eng, model, 0).predict(Rq)
            _same('M = 16385 at 5 slices vs 0: F', F, F0)


def test_slice_argument_limits(eng):
    """1 and 8 slices are argument errors; on a D <= 256 model every setting leaves the fused kernel bit-identical."""
    model, _, _ = opm.make_model(24, 29, 'plain', seed=0)
    p = eng.GDMLPredict(model)
    for bad in (1, 8):
        with pytest.raises(Exception):
            p.set_contraction_slices(bad)
    small, _, _ = opm.make_model(22, 29, 'plain', seed=0)  # D = 231
    Rq = opm.queries(small, 3, seed=1)
    E0, F0 = eng.GDMLPredict(small).predict(Rq)
    ps = eng.GDMLPredict(small)
    ps.set_contraction_slices(5)
    E5, F5 = ps.predict(Rq)
    _same('D <= 256 with 5 slices: F', F5, F0)
    _same('D <= 256 with 5 slices: E', E5, E0)


def test_report_against_documented(eng):
    """Prints the observed force error per slice count (from test_stages_and_end_to_end) beside the documented one."""
    if not _REPORT:
        pytest.skip('run with test_stages_and_end_to_end')
    for S in SLICES:
        vals = [v for (kind, s), v in _REPORT.items() if s == S]
        if vals:
            print('S=%d: observed max rel err %.2e, documented %s' % (S, max(vals), DOCUMENTED.get(S, '-')))


# ------------------------------------------------------------------------------------------------ c. call paths
@pytest.mark.parametrize('kind', opm.KINDS)
def test_call_paths_bit_identical(eng, kind):
    """Rows are independent (each row of every operand is split with its own exponent), so every route gives the tapped
    single-chunk rows bit for bit."""
    import torch

    from sgdml_b200 import _lib

    model, R, g, _, _, _ = _case(kind)
    M = R.shape[0]
    Rq = opm.queries(model, 9, seed=11)
    p = _predictor(eng, model, 5, R_d_desc=g)
    t, arr, E, F = tapped(p, model, R=Rq)
    for rep in range(2):  # capture, then replay
        Eh, Fh = p.predict(Rq[:5])
        _same('host <= 16 (graph, pass %d): F' % rep, Fh, F[:5])
        _same('host <= 16 (graph, pass %d): E' % rep, Eh, E[:5])
    Ed, Fd = p.predict(torch.from_numpy(Rq).cuda())
    _same('device tensors: F', Fd.cpu().numpy(), F)
    _same('device tensors: E', Ed.cpu().numpy(), E)
    Ev, Fv, Wv = p.predict_virial(Rq)
    _same('predict_virial: F', Fv, F)
    _same('predict_virial: E', Ev, E)
    if 'lattice' in model:
        cells = np.repeat(np.asarray(model['lattice'])[None], Rq.shape[0], axis=0)
        Ec, Fc, Wc = p.predict_virial(Rq, lattice=cells)
        _same('predict_virial_cells: F', Fc, F)
        _same('predict_virial_cells: E', Ec, E)
    # training points: predict(R=None) (scaled) and K.v over an odd range (raw sums)
    tt, _, Et, Ft = tapped(p, model, n_geo=M, m_begin=0, scaled=1, stages=False)
    Er, Fr = p.predict()
    _same('predict(R=None): F', Fr, Ft)
    _same('predict(R=None): E', Er, Et)
    _, _, Ek, Fk = tapped(p, model, n_geo=13, m_begin=3, scaled=0, stages=False)
    E_out = np.empty(13)
    _same('kmatvec_train [3, 16): F', p.kmatvec_train(3, 16, E_out=E_out), Fk)
    _same('kmatvec_train [3, 16): E', E_out, Ek)
    # chunk caps 1 and 7 (applied to models created after the call)
    for cap in (1, 7):
        _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(cap), 'set_predict_chunk')
        try:
            pc_ = _predictor(eng, model, 5)
            Ec_, Fc_ = pc_.predict(torch.from_numpy(Rq).cuda())
        finally:
            _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(0), 'set_predict_chunk')
        _same('chunk cap %d: F' % cap, Fc_.cpu().numpy(), F)
        _same('chunk cap %d: E' % cap, Ec_.cpu().numpy(), E)


def test_pipelined_host_queries_bit_identical(eng):
    """>= 4096 pinned host queries run pipelined over workspace slots 0 and 1: bit-identical to the device-tensor call
    (itself one chunk, the tapped rows by the test above)."""
    import torch

    model, _, _ = opm.make_model(24, 29, 'perms', seed=5)
    Rq = opm.queries(model, 4500, seed=6)
    p = _predictor(eng, model, 5)
    Ed, Fd = p.predict(torch.from_numpy(Rq).cuda())
    Ep, Fp = p.predict(torch.from_numpy(Rq).pin_memory())
    _same('pipelined pinned host: F', Fp.numpy(), Fd.cpu().numpy())
    _same('pipelined pinned host: E', Ep.numpy(), Ed.cpu().numpy())


# ------------------------------------------------------------------------------------------------ d. model state
def _batch(p, Rq):
    """A graph-replayed host batch (second call of its size) and a device-tensor batch."""
    import torch

    p.predict(Rq[:3])
    Eh, Fh = p.predict(Rq[:3])
    Ed, Fd = p.predict(torch.from_numpy(Rq).cuda())
    return Eh, Fh, Ed.cpu().numpy(), Fd.cpu().numpy()


def _assert_state(what, got, want):
    for name, a, b in zip(('E graph', 'F graph', 'E device', 'F device'), got, want):
        _same('%s: %s' % (what, name), a, b)


def test_model_state_transitions(eng, monkeypatch):
    from sgdml_b200 import _lib
    from oracle import desc as odesc

    model, R, g, _, _, _ = _case('ecstr')
    M, N = R.shape[0], 24
    Rq = opm.queries(model, 6, seed=21)
    rng = np.random.default_rng(8)
    v1, v2 = rng.standard_normal(M * 3 * N), rng.standard_normal(M * 3 * N)
    aE = model['alphas_E']
    plain = {k: v for k, v in model.items() if k != 'alphas_E'}

    def fresh(S, alphas, with_E=True, R_d_desc=g, base=model):
        p = _predictor(eng, base if with_E else plain, S, R_d_desc=R_d_desc)
        p.set_alphas(alphas)
        return _batch(p, Rq)

    p = _predictor(eng, model, 5, R_d_desc=g)
    _batch(p, Rq)
    p.set_alphas(v1)
    p.set_alphas(v2)
    _assert_state('set_alphas twice', _batch(p, Rq), fresh(5, v2))
    _lib.check(_lib.lib().sgdml_b200_model_set_alphas_E(p._handle, None, _lib.current_stream()), 'set_alphas_E')
    _assert_state('set_alphas_E off', _batch(p, Rq), fresh(5, v2, with_E=False))
    p._set_alphas_E(aE)
    _assert_state('set_alphas_E on', _batch(p, Rq), fresh(5, v2))
    _, g2 = odesc.from_R(opm.queries(model, M, seed=31))
    p.set_R_d_desc(g2)
    p.set_alphas(v1)
    _assert_state('set_R_d_desc', _batch(p, Rq), fresh(5, v1, R_d_desc=g2))
    for S in (6, 0, 5):
        p.set_contraction_slices(S)
        _assert_state('slices -> %d' % S, _batch(p, Rq), fresh(S, v1, R_d_desc=g2))
    monkeypatch.setenv('SGDML_B200_OZAKI_PREDICT_SLICES', '5')
    pe = eng.GDMLPredict(model)
    pe.set_R_d_desc(g2)
    pe.set_alphas(v1)
    monkeypatch.delenv('SGDML_B200_OZAKI_PREDICT_SLICES')
    _assert_state('created under SGDML_B200_OZAKI_PREDICT_SLICES=5', _batch(pe, Rq), fresh(5, v1, R_d_desc=g2))


def test_set_lattice_transition(eng):
    """set_lattice on a periodic model at 5 slices: bit-identical to a fresh model created in the new cell."""
    from sgdml_b200 import _lib

    model, _, _, _, _, _ = _case('pbc')
    Rq = opm.queries(model, 6, seed=23)
    p = _predictor(eng, model, 5)
    _batch(p, Rq)
    lat2 = np.ascontiguousarray(np.asarray(model['lattice']) * 1.07)
    _lib.check(_lib.lib().sgdml_b200_model_set_lattice(p._handle, _lib.ptr(lat2),
                                                       _lib.ptr(np.ascontiguousarray(np.linalg.inv(lat2)))),
               'set_lattice')
    m2 = dict(model, lattice=lat2)
    _assert_state('set_lattice', _batch(p, Rq), _batch(_predictor(eng, m2, 5), Rq))
