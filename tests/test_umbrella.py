"""Umbrella sampling with replica exchange on the device (sgdml_b200_umbrella_*, sgdml_b200.GDMLUmbrellaSampling)
against the NumPy restatement of tests/umbrella_oracle.py, fed by the engine's predictor on device-resident positions.

GPU: trajectories, CVs, restraint energies, walker labels and acceptance counts against the restatement on two MD
fixtures; zero force constants against sgdml_b200_md_run; graph against plain launches and chunks; continuation,
set_windows, isolation; the handle-kind rules of the new kind and bad input; the public units; MBAR against the NumPy
MBAR; and the physics of a trained double well: the profile from REUS and MBAR against unbiased sampling.
"""

import ctypes

import numpy as np
import pytest

import metad_oracle as mo
import umbrella_oracle as uo
from conftest import rel_err
from md_common import _cuda_forces, md_fs_masses

pytestmark = pytest.mark.gpu

CVS = [('distance', (0, 1)), ('angle', (1, 2, 3)), ('dihedral', (0, 2, 3, 4))]
NL, NW = 2, 4  # ladders, windows


def _setup(name, chunk=0, scale=1.0, shift=0.0):
    """(GDMLPredict, GDMLUmbrellaSampling in model units, R0, V0, dt, (gamma, kT))"""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    Rc = np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)
    gp = sgdml_b200.GDMLPredict(model)
    N = gp.n_atoms
    masses = md_fs_masses(np.linspace(1.0, 16.0, N))
    n = NL * NW
    R0 = Rc[np.arange(n) % Rc.shape[0]]
    _, F0 = gp.predict(R0[:1])
    s0 = np.array([mo.cv_eval(k, a, R0[:1].reshape(1, -1, 3))[0][0] for k, a in CVS])
    steps = np.array([0.02, 0.05, 0.1])
    centers = s0[None] + (np.arange(NW)[:, None] - 1.5 + shift) * steps[None]
    centers[:, 2] = mo.wrap(centers[:, 2])
    centers[:, 2] = np.where(centers[:, 2] == -np.pi, np.pi, centers[:, 2])
    # restraint forces a sizeable share of the model's: kappa steps about a fifth of max |F|
    kappas = np.tile(scale * 0.2 * float(np.max(np.abs(F0))) / steps, (NW, 1))
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        dyn = sgdml_b200.GDMLUmbrellaSampling(gp, masses, CVS, centers, kappas, n_ladders=NL, E_to_eV=1.0,
                                              F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    s = dyn.inv_mass.repeat(3)
    dt = float(np.sqrt(2e-3 / max(np.max(np.abs(F0 * s)), 1e-300)))
    V0 = np.random.default_rng(2).standard_normal(R0.shape) * 1e-3 / dt
    kT = float(np.mean(V0 * V0 / s))
    return gp, dyn, R0, V0, dt, (0.1 / dt, kT)


def _same(a, b):
    return set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize('name', ['n9_m16_s6', 'pbc_n6_m8'])
def test_matches_restatement(name):
    gp, dyn, R0, V0, dt, (gamma, kT) = _setup(name)
    start, n, seed, every = (1 << 32) - 25, 60, (9 << 32) + 4, 3
    dyn._set_state_raw(R0, V0, step=start)
    fr = dyn._run_raw(n, dt, gamma, kT, every, seed=seed, stride=1)
    s = dyn.inv_mass.repeat(3)
    forces = _cuda_forces(gp)
    C, K = dyn._raw_windows(*dyn.windows)
    h, c1, sigma = mo.md_oracle.constants(dt, gamma, kT, s)
    stats = {'n_accepted': np.zeros((NL, NW - 1), dtype=np.int64),
             'n_attempted': np.zeros((NL, NW - 1), dtype=np.int64), 'margin': np.inf}
    worst = {}
    # Each step restated from the device's frame before it (CUDA's exp and atan2 may differ from NumPy's in the last
    # bit; the tolerances are metadynamics' and for the same reasons: tests/test_metad.py).
    for f in range(n):
        c = start + f + 1
        Rp, Vp, Wp = (R0, V0, np.arange(NL * NW)) if f == 0 else (fr['R'][f - 1], fr['V'][f - 1], fr['walker'][f - 1])
        st = {'R': np.array(Rp), 'V': np.array(Vp), 'walker': np.array(Wp, dtype=np.int32)}
        uo.evaluate(st, forces, CVS, C, K)
        Vh = st['V'] + h * (st['F'] * s)
        st['R'] = st['R'] + h * Vh
        Vh = c1 * Vh + sigma * mo.md_oracle.normals(seed, c - 1, Vh.shape[0], Vh.shape[1])
        st['R'] = st['R'] + h * Vh
        uo.evaluate(st, forces, CVS, C, K)
        st['V'] = Vh + h * (st['F'] * s)
        if uo.remd_oracle.is_exchange(c, start, every):
            uo.exchange(st, c, every, seed, 1.0 / kT, h, s, CVS, C, K, stats)
        assert np.array_equal(fr['walker'][f], st['walker']), f
        for k, ref in (('R', st['R']), ('V', st['V']), ('E_pot', st['E']), ('E_kin', mo.md_oracle.kinetic(st['V'], s)),
                       ('cv', st['cv']), ('bias', st['bias'])):
            e = rel_err(fr[k][f], ref)
            worst[k] = max(worst.get(k, 0.0), e)
            assert e < (1e-9 if k in ('V', 'E_pot', 'E_kin', 'bias') else 1e-11), (f, k, e)
        # the CV frames are the CVs of the R frames; the walker frames are permutations within each ladder
        X = fr['R'][f].reshape(NL * NW, -1, 3)
        assert rel_err(fr['cv'][f], np.stack([mo.cv_eval(k, a, X)[0] for k, a in CVS], 1)) < 1e-12
        for l in range(NL):
            assert sorted(fr['walker'][f][l * NW:(l + 1) * NW]) == list(range(l * NW, (l + 1) * NW))
    print('%s: worst per-step deviation %s, accepted %s of %s, smallest |u - exp(d)| %.3g'
          % (name, worst, fr['n_accepted'].tolist(), fr['n_attempted'].tolist(), stats['margin']))
    assert np.array_equal(fr['n_attempted'], stats['n_attempted'])
    assert np.array_equal(fr['n_accepted'], stats['n_accepted'])
    assert fr['n_accepted'].sum() > 0
    assert np.array_equal(fr['walkers'], fr['walker'][-1])
    sd = dyn._get_state_raw()
    assert np.array_equal(sd['R'], fr['R'][-1]) and np.array_equal(sd['E_pot'], fr['E_pot'][-1])
    assert np.array_equal(sd['F'], forces(sd['R'])[1])  # get_state's F is the model's
    b = dyn._get_bias_raw()
    assert np.array_equal(b['cv'], fr['cv'][-1]) and np.array_equal(b['V'], fr['bias'][-1])


def test_zero_force_constants_without_exchange_is_md_run():
    import sgdml_b200

    gp, dyn, R0, V0, dt, (gamma, kT) = _setup('n9_m16_s6', scale=0.0)
    md = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), n_replicas=NL * NW,
                                 E_to_eV=1.0, F_to_eV_Ang=1.0)
    dyn._set_state_raw(R0, V0, step=11)
    md._set_state_raw(R0, V0, step=11)
    a = dyn._run_raw(30, dt, gamma, kT, 0, seed=3, stride=10)
    b = md._run_raw(30, dt, gamma, kT, seed=3, stride=10)
    for k in ('R', 'V', 'E_pot', 'E_kin'):
        assert np.array_equal(a[k], b[k]), k
    assert np.all(a['bias'] == 0.0) and np.all(a['walker'] == np.arange(NL * NW))
    assert _same(dyn._get_state_raw(), md._get_state_raw())


def _run(d, R0, V0, dt, args, n=24, seed=8):
    d._set_state_raw(R0, V0)
    out = d._run_raw(n, dt, *args, 3, seed=seed, stride=4)
    return out, d._get_state_raw(), d._get_bias_raw()


def test_graph_matches_plain_launches_and_chunks(monkeypatch):
    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')
    a = _run(dyn, R0, V0, dt, args)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _run(dyn, R0, V0, dt, args)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    _, dc, _, _, _, _ = _setup('n9_m16_s6', chunk=2)
    c = _run(dc, R0, V0, dt, args)
    assert a[0]['n_accepted'].sum() > 0
    for x in (b, c):
        assert all(_same(u, v) for u, v in zip(a, x))


def test_continuation_set_windows_and_isolation():
    import torch

    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')
    _, dyn2, _, _, _, _ = _setup('n9_m16_s6')
    _, moved, _, _, _, _ = _setup('n9_m16_s6', shift=0.5, scale=2.0)
    for d in (dyn, dyn2):
        d._set_state_raw(R0, V0, step=5)
    a = dyn._run_raw(40, dt, *args, 3, seed=99, stride=5)
    b1 = dyn2._run_raw(20, dt, *args, 3, seed=99, stride=5)
    # predict calls and another umbrella handle between the halves change nothing
    Rbig = np.tile(R0, (12, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((96, R0.shape[1]))
    gp.predict(Rbig)
    gp.predict(torch.from_numpy(Rbig).cuda())
    moved._set_state_raw(R0 + 0.01, V0)
    moved._run_raw(9, dt, *args, 2, seed=2)
    b2 = dyn2._run_raw(20, dt, *args, 3, seed=99, stride=5)
    frames = [k for k in a if k not in ('walkers', 'n_accepted', 'n_attempted')]
    assert _same({k: a[k] for k in frames}, {k: np.concatenate([b1[k], b2[k]]) for k in frames})
    assert np.array_equal(a['n_accepted'], b1['n_accepted'] + b2['n_accepted'])
    assert np.array_equal(a['walkers'], b2['walkers'])
    # set_windows: the state's restraints are re-evaluated, and a run goes on as on a handle made with those windows
    st = dyn._get_state_raw()
    dyn.set_windows(*moved.windows)
    moved._set_state_raw(st['R'], st['V'], step=st['step'])
    dyn._set_state_raw(st['R'], st['V'], step=st['step'])
    assert _same(dyn._get_bias_raw(), moved._get_bias_raw())
    assert _same(dyn._run_raw(12, dt, *args, 3, seed=4, stride=4), moved._run_raw(12, dt, *args, 3, seed=4, stride=4))


def test_handle_kind_rules_and_bad_input():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, dyn, R0, V0, dt, (gamma, kT) = _setup('n9_m16_s6')
    L = _lib.lib()
    st = _lib.current_stream()
    inv_mass = dyn.inv_mass
    C, K = dyn._raw_windows(*dyn.windows)
    types = np.array([0, 1, 2], dtype=np.int32)
    atoms = np.array([[0, 1, 0, 0], [1, 2, 3, 0], [0, 2, 3, 4]], dtype=np.int64)
    h = ctypes.c_void_p()
    bad_c, bad_k = C.copy(), K.copy()
    bad_c[0, 2] = 4.0
    for c, k in ((bad_c, K), (C, -K), (C * np.nan, K), (C, K * np.inf)):
        c, k = np.ascontiguousarray(c), np.ascontiguousarray(k)
        assert L.sgdml_b200_umbrella_create(ctypes.byref(h), gp._handle, NL, NW, inv_mass.ctypes.data, 3,
                                            types.ctypes.data, atoms.ctypes.data, c.ctypes.data,
                                            k.ctypes.data) <= -1000 and not h.value
    with pytest.raises(_lib.EngineError):
        dyn._run_raw(6, dt, gamma, kT)  # no state yet
    with pytest.raises(_lib.EngineError):
        dyn._get_bias_raw()
    dyn._set_state_raw(R0, V0, step=7)
    dyn._run_raw(6, dt, gamma, kT, 2, seed=1)
    H = dyn._handle
    before = dyn._get_state_raw(), dyn._get_bias_raw()
    for bad in (dict(kT=0.0, every=2), dict(every=-1), dict(gamma=np.nan), dict(stride=4), dict(dt=0.0)):
        kw = dict(dict(kT=kT, every=2, gamma=gamma, stride=0, dt=dt), **bad)
        out = {k: np.full((6, NL * NW, 27), 1.5) for k in ('R', 'cv')}
        rc = L.sgdml_b200_umbrella_run(H, 6, kw['dt'], kw['gamma'], kw['kT'], 0, kw['every'], kw['stride'],
                                       out['R'].ctypes.data, None, None, None, out['cv'].ctypes.data, None, None, None,
                                       None, None, st)
        assert rc <= -1000, bad
        assert np.all(out['R'] == 1.5) and np.all(out['cv'] == 1.5)
    assert L.sgdml_b200_umbrella_set_windows(H, np.ascontiguousarray(bad_c).ctypes.data, K.ctypes.data, st) <= -1000
    # the kinds: every other entry point refuses an umbrella handle, and the umbrella ones refuse the other kinds
    R = np.zeros((6, NL * NW, 27))
    assert L.sgdml_b200_md_run(H, 6, dt, gamma, kT, 0, 0, None, None, None, None, st) <= -1000
    ktab = np.full(NW, kT)
    assert L.sgdml_b200_remd_run(H, NW, ktab.ctypes.data, 6, dt, gamma, 0, 2, 0, None, None, None, None, None, None,
                                 None, None, st) <= -1000
    assert L.sgdml_b200_pimd_run(H, 6, dt, kT, 1.0, gamma, 1.0, 0, 0, None, None, None, None, None, None, st) <= -1000
    w = np.full(3, 0.1)
    assert L.sgdml_b200_metad_run(H, 6, dt, gamma, kT, 0.1, w.ctypes.data, 2, 1.0, 0, 0, None, None, None, None, None,
                                  None, st) <= -1000
    assert L.sgdml_b200_metad_get_bias(H, None, None, None, st) <= -1000
    n_out = np.zeros(NL * NW, dtype=np.int64)
    assert L.sgdml_b200_relax_fire(H, 5, 0.1, 0.1, 0.1, 1.0, n_out.ctypes.data, None, None, st) <= -1000
    assert L.sgdml_b200_relax_lbfgs(H, 5, 0.1, 0.1, 5, 1.0, n_out.ctypes.data, None, None, st) <= -1000
    assert L.sgdml_b200_neb_fire(H, NW, 5, 0.1, 1.0, 0, 0.1, 0.1, 1.0, n_out.ctypes.data, None, None, None,
                                 st) <= -1000
    modes = np.ones((NL * NW // 2, 27))
    assert L.sgdml_b200_dimer_fire(H, modes.ctypes.data, 5, 0.1, 1e-3, 0.7071067811865476, 0.7071067811865476, 0.0,
                                   0.1, 0.1, 1.0, n_out.ctypes.data, None, None, None, None, None, st) <= -1000
    assert L.sgdml_b200_npt_run(H, 6, dt, gamma, kT, 0.0, 1.0, 100.0, 0, 0, R.ctypes.data, None, None, None, None,
                                None, st) <= -1000
    assert L.sgdml_b200_npt_get_cells(H, R.ctypes.data, None, None, st) <= -1000
    assert L.sgdml_b200_metad_get_hills(H, n_out.ctypes.data, None, None, None, st) <= -1000
    assert np.all(R == 0.0) and np.all(n_out == 0)
    after = dyn._get_state_raw(), dyn._get_bias_raw()
    assert _same(before[0], after[0]) and _same(before[1], after[1])
    plain = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), n_replicas=NL * NW,
                                    E_to_eV=1.0, F_to_eV_Ang=1.0)
    plain._set_state_raw(R0, V0)
    P = plain._handle
    assert L.sgdml_b200_umbrella_run(P, 6, dt, gamma, kT, 0, 0, 0, None, None, None, None, None, None, None, None,
                                     None, None, st) <= -1000
    assert L.sgdml_b200_umbrella_get_bias(P, None, None, None, st) <= -1000
    assert L.sgdml_b200_umbrella_set_windows(P, C.ctypes.data, K.ctypes.data, st) <= -1000
    meta = sgdml_b200.GDMLMetadynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), CVS, n_walkers=NL * NW,
                                       E_to_eV=1.0, F_to_eV_Ang=1.0)
    meta._set_state_raw(R0, V0)
    assert L.sgdml_b200_umbrella_run(meta._handle, 6, dt, gamma, kT, 0, 0, 0, None, None, None, None, None, None, None,
                                     None, None, None, st) <= -1000
    assert L.sgdml_b200_umbrella_get_bias(meta._handle, None, None, None, st) <= -1000
    with pytest.raises(ValueError):
        sgdml_b200.GDMLUmbrellaSampling(gp, md_fs_masses(np.ones(gp.n_atoms)), CVS, C[:, :2], K[:, :2])


def test_public_units():
    """GDMLUmbrellaSampling in eV / Angstrom / fs with a kcal/mol model against the raw calls in model units; torch in,
    torch out; MBAR and the profile through the public interface."""
    import torch

    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc
    from sgdml_b200.md import KB_EV

    gp, raw, R0, V0, dt, (gamma, kT) = _setup('n9_m16_s6')
    masses = md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms))
    C, K = raw.windows
    pub = sgdml_b200.GDMLUmbrellaSampling(gp, masses * kc, CVS, C, K * kc, n_ladders=NL)  # the same inverse masses
    assert np.allclose(pub.inv_mass, raw.inv_mass, rtol=1e-15)
    T = kT * kc / KB_EV
    raw._set_state_raw(R0, V0)
    a = raw._run_raw(12, dt, gamma, kT, 3, seed=4, stride=4)
    pub.set_state(torch.from_numpy(R0.reshape(NL, NW, -1, 3)).cuda(), torch.from_numpy(V0).cuda().reshape(NL, NW, -1, 3))
    b = pub.run(12, dt, T, gamma, exchange_every=3, seed=4, stride=4)
    assert isinstance(b['cv'], torch.Tensor) and b['cv'].shape == (3, NL, NW, 3)
    assert rel_err(b['positions'].cpu().numpy().reshape(a['R'].shape), a['R']) < 1e-13
    assert rel_err(b['cv'].cpu().numpy().reshape(a['cv'].shape), a['cv']) < 1e-13
    assert rel_err(b['bias_energy'].cpu().numpy().ravel() / kc, a['bias'].ravel()) < 1e-12
    assert np.array_equal(b['walker'].cpu().numpy().reshape(a['walker'].shape), a['walker'])
    s = pub.get_state()
    rb = raw._get_bias_raw()
    assert s['cv'].shape == (NL, NW, 3) and s['bias_forces'].shape == (NL, NW, gp.n_atoms, 3)
    assert rel_err(s['bias_forces'].cpu().numpy().reshape(rb['F'].shape) / kc, rb['F']) < 1e-12
    m_pub = pub.mbar(b['cv'], T)
    m_np = raw.mbar(a['cv'].reshape(3, NL, NW, 3), kT / KB_EV)  # raw: E_to_eV = 1, so eV are model units
    for x, y in zip(m_pub, m_np):
        assert rel_err(x['f'].cpu().numpy() / kc, y['f']) < 1e-9
        assert isinstance(x['log_w'], torch.Tensor) and x['log_w'].shape == (3, NW)
    fe = pub.free_energy(b['cv'], np.linspace(C[0, 0] - 0.05, C[-1, 0] + 0.05, 5), T)
    assert isinstance(fe, torch.Tensor) and fe.shape == (NL, 4)
    assert np.nanmin(fe.cpu().numpy()) == 0.0


def test_mbar_against_numpy():
    """umbrella_mbar against the NumPy MBAR of tests/umbrella_oracle.py on two CVs (a distance and a dihedral across
    +-pi), host and device inputs, the same bits on every call; one window gives f = 0."""
    import torch

    from sgdml_b200 import _lib

    _, dyn, _, _, _, _ = _setup('n9_m16_s6')
    rng = np.random.default_rng(3)
    K, n_k = 6, 3000
    c = np.stack([np.linspace(1.0, 1.5, K), np.linspace(2.6, 3.1, K)], 1)
    c[:, 1] = mo.wrap(c[:, 1])
    kap = np.stack([np.full(K, 200.0), np.full(K, 40.0)], 1)
    beta = 2.0
    S = np.concatenate([np.stack([ck[0] + rng.standard_normal(n_k) / np.sqrt(beta * kap[0, 0]),
                                  mo.wrap(ck[1] + rng.standard_normal(n_k) / np.sqrt(beta * kap[0, 1]))], 1)
                        for ck in c])
    types = ['distance', 'dihedral']
    u = np.array([beta * uo.restraint(S, types, c[k], kap[k])[0] for k in range(K)])
    f_ref, lw_ref, it_ref = uo.mbar(u, [n_k] * K, tol=1e-12)
    L = _lib.lib()
    tt = np.array([0, 2], dtype=np.int32)
    counts = np.full(K, n_k, dtype=np.int64)

    def call(samples, f, lw):
        n_iter, resid = np.zeros(1, dtype=np.int64), np.zeros(1)
        _lib.check(L.sgdml_b200_umbrella_mbar(K, 2, tt.ctypes.data, c.ctypes.data, kap.ctypes.data, beta, K * n_k,
                                              _lib.ptr(samples), counts.ctypes.data, 1e-12, 10000, _lib.ptr(f),
                                              _lib.ptr(lw), n_iter.ctypes.data, resid.ctypes.data,
                                              _lib.current_stream()), 'mbar')
        return int(n_iter[0]), float(resid[0])

    f1, lw1 = np.empty(K), np.empty(K * n_k)
    it1, r1 = call(S, f1, lw1)
    f2, lw2 = np.empty(K), np.empty(K * n_k)
    call(S, f2, lw2)
    Sd = torch.from_numpy(S).cuda()
    f3, lw3 = torch.empty(K, dtype=torch.float64, device='cuda'), torch.empty(K * n_k, dtype=torch.float64, device='cuda')
    it3, _ = call(Sd, f3, lw3)
    print('MBAR: %d iterations (NumPy %d), resid %.3g, max |f - f_numpy| %.3g' % (it1, it_ref, r1,
                                                                                 np.max(np.abs(f1 - f_ref))))
    assert np.array_equal(f1, f2) and np.array_equal(lw1, lw2)
    assert np.array_equal(f1, f3.cpu().numpy()) and np.array_equal(lw1, lw3.cpu().numpy()) and it1 == it3
    assert r1 < 1e-12 and abs(it1 - it_ref) <= 2
    assert np.max(np.abs(f1 - f_ref)) < 1e-9 and np.max(np.abs(lw1 - lw_ref)) < 1e-9
    assert abs(np.exp(lw1).sum() - 1.0) < 1e-12
    # one window: f = 0, one iteration
    f1w, lw1w = np.empty(1), np.empty(n_k)
    n1 = np.array([n_k], dtype=np.int64)
    it, resid = np.zeros(1, dtype=np.int64), np.zeros(1)
    _lib.check(L.sgdml_b200_umbrella_mbar(1, 2, tt.ctypes.data, c.ctypes.data, kap.ctypes.data, beta, n_k,
                                          S.ctypes.data, n1.ctypes.data, 1e-12, 100, f1w.ctypes.data,
                                          lw1w.ctypes.data, it.ctypes.data, resid.ctypes.data, 0), 'mbar')
    assert f1w[0] == 0.0 and it[0] == 1
    # bad input: non-finite samples, counts that do not add up
    bad = S.copy()
    bad[5, 1] = np.nan
    for smp, cnt in ((bad, counts), (S, counts + 1)):
        assert L.sgdml_b200_umbrella_mbar(K, 2, tt.ctypes.data, c.ctypes.data, kap.ctypes.data, beta, K * n_k,
                                          smp.ctypes.data, cnt.ctypes.data, 1e-12, 100, f1w.ctypes.data, None, None,
                                          None, 0) <= -1000


# ---------------------------------------------------------------------------------------------------- physics
def _d01(R):
    X = np.asarray(R).reshape(-1, 4, 3)
    return np.linalg.norm(X[:, 0] - X[:, 1], axis=-1)


def test_reus_profile_matches_unbiased_sampling():
    """At kT = 0.04 (barrier 2.5 kT) unbiased Langevin of 64 replicas crosses often, and -kT ln of its d01 histogram is
    the free-energy profile.  Four ladders of 16 umbrella windows along d01 with exchanges, reweighted by MBAR, give the
    same well-to-well free-energy difference and barrier within four standard errors across ladders plus 0.25 kT,
    and every neighbour pair exchanges."""
    import sgdml_b200
    from test_metad import _dw_model
    from sgdml_b200.md import KB_EV
    from test_neb import _DW_DC, _DW_HI, _DW_LO, _DW_PHI, _dw_hinge

    gp = _dw_model()
    kT, dt, gamma = 0.04, 0.02, 1.0
    masses = md_fs_masses(np.ones(4))
    A = _dw_hinge(_DW_PHI[0]).reshape(1, 12)
    B = _dw_hinge(_DW_PHI[1]).reshape(1, 12)
    md = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=64, E_to_eV=1.0, F_to_eV_Ang=1.0)
    md._set_state_raw(np.concatenate([np.tile(A, (32, 1)), np.tile(B, (32, 1))]))
    md._run_raw(2000, dt, gamma, kT, seed=1)
    d_unb = _d01(md._run_raw(40000, dt, gamma, kT, seed=2, stride=20, frames=('R',))['R'])
    edges = np.linspace(np.quantile(d_unb, 0.002), np.quantile(d_unb, 0.998), 31)
    mid = 0.5 * (edges[1:] + edges[:-1])
    p, _ = np.histogram(d_unb, edges)
    F_unb = -kT * np.log(np.maximum(p, 1) / p.max())

    n_lad, n_win = 4, 16
    lo, hi = _DW_LO - 0.1, _DW_HI + 0.1
    centers = np.linspace(lo, hi, n_win)
    kappa = kT / ((hi - lo) / (n_win - 1)) ** 2  # one thermal width per window spacing
    us = sgdml_b200.GDMLUmbrellaSampling(gp, masses, [('distance', (0, 1))], centers, np.full(n_win, kappa),
                                         n_ladders=n_lad, E_to_eV=1.0, F_to_eV_Ang=1.0)
    phi = np.linspace(_DW_PHI[0] - 0.1, _DW_PHI[1] + 0.1, n_win)
    us._set_state_raw(np.tile(_dw_hinge(phi).reshape(n_win, 12), (n_lad, 1)))
    us._run_raw(2000, dt, gamma, kT, 10, seed=3)
    fr = us._run_raw(20000, dt, gamma, kT, 10, seed=4, stride=10, frames=('cv', 'walker'))
    acc = fr['n_accepted'] / fr['n_attempted']
    print('REUS acceptance per pair: min %.3f, mean %.3f' % (acc.min(), acc.mean()))
    assert np.all(fr['n_accepted'] > 0)
    cv = fr['cv'].reshape(-1, n_lad, n_win, 1)
    F_us = us.free_energy(cv, edges, kT / KB_EV)  # (n_lad, bins), model units (E_to_eV = 1)

    def summary(F):
        ok = np.isfinite(F)
        left, right = (mid < _DW_DC) & ok, (mid > _DW_DC) & ok
        fl = -kT * np.log(np.exp(-F[left] / kT).sum())
        fr_ = -kT * np.log(np.exp(-F[right] / kT).sum())
        between = (mid > mid[left][np.argmin(F[left])]) & (mid < mid[right][np.argmin(F[right])]) & ok
        return fr_ - fl, F[between].max() - min(F[left].min(), F[right].min())

    ref = summary(F_unb)
    per = np.array([summary(f) for f in F_us])
    mean, sem = per.mean(0), per.std(0, ddof=1) / np.sqrt(n_lad)
    tol = 4.0 * sem + 0.25 * kT
    print('unbiased dF %.4f barrier %.4f; REUS + MBAR dF %.4f +- %.4f, barrier %.4f +- %.4f (kT %.3f)'
          % (ref[0], ref[1], mean[0], sem[0], mean[1], sem[1], kT))
    assert np.all(np.abs(mean - np.array(ref)) < tol), (mean, ref, tol)
