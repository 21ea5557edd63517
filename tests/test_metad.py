"""Multiple-walker metadynamics on the device (sgdml_b200_metad_*, sgdml_b200.GDMLMetadynamics) against the NumPy
restatement of tests/metad_oracle.py, fed by the engine's predictor on device-resident positions.

GPU: trajectories, CVs, bias energies and hills against the restatement on two MD fixtures, zero height against
sgdml_b200_md_run, graph against plain launches and chunks, continuation and restarts from the hills, isolation from
the predictor's calls and from other handles, bad input, the public units, and the physics of a trained double well:
barrier crossing at low temperature and the free-energy profile against unbiased sampling.  Which entry points take a
metadynamics handle is tests/test_md_handle_kinds.py's.
"""

import ctypes

import numpy as np
import pytest

import metad_oracle as mo
from conftest import rel_err
from md_common import _cuda_forces, md_fs_masses

pytestmark = pytest.mark.gpu

CVS = [('distance', (0, 1)), ('angle', (1, 2, 3)), ('dihedral', (0, 2, 3, 4)), ('dihedral', (4, 3, 1, 5))]
NW, NG = 2, 3  # walkers per group, groups


def _setup(name, n_cv=4, chunk=0, nw=NW, ng=NG):
    """(GDMLPredict, GDMLMetadynamics in model units, R0, V0, dt, run arguments (gamma, kT, w0, widths, pace, dkT))."""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    Rc = np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)
    gp = sgdml_b200.GDMLPredict(model)
    N = gp.n_atoms
    masses = md_fs_masses(np.linspace(1.0, 16.0, N))
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        dyn = sgdml_b200.GDMLMetadynamics(gp, masses, CVS[:n_cv], n_walkers=nw, n_groups=ng, E_to_eV=1.0,
                                          F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    n = nw * ng
    R0 = Rc[np.arange(n) % Rc.shape[0]]
    _, F0 = gp.predict(R0[:1])
    s = dyn.inv_mass.repeat(3)
    dt = float(np.sqrt(2e-3 / max(np.max(np.abs(F0 * s)), 1e-300)))
    V0 = np.random.default_rng(2).standard_normal(R0.shape) * 1e-3 / dt
    kT = float(np.mean(V0 * V0 / s))
    widths = np.array([0.02, 0.05, 0.05, 0.05])[:n_cv]
    # hills whose force is a sizeable share of the model's: w0 / width about a fifth of max |F|
    w0 = 0.2 * float(np.max(np.abs(F0))) * 0.02
    return gp, dyn, R0, V0, dt, (0.1 / dt, kT, w0, widths, 3, 4.0 * w0)


def _hills_before(hills_dev, count0, c, start, pace, nw):
    """the device's hills of each group committed before state c of a run from `start`"""
    n, C, W, H = hills_dev
    edges = np.concatenate([[0], np.cumsum(n)])
    k = 0 if c <= start else (c - 1) // pace - start // pace
    out = []
    for g in range(len(n)):
        m = count0[g] + nw * k
        a = edges[g]
        out.append((C[a:a + m], W[a:a + m], H[a:a + m]))
    return out


def _same(a, b):
    return set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize('name', ['n9_m16_s6', 'pbc_n6_m8'])
def test_matches_restatement(name):
    gp, dyn, R0, V0, dt, args = _setup(name)
    gamma, kT, w0, widths, pace, dkT = args
    start, n, seed = (1 << 32) - 25, 60, (9 << 32) + 4  # the counter crosses 2^32 inside the run
    dyn._set_state_raw(R0, V0, step=start)
    b0 = dyn._get_bias_raw()
    assert np.all(b0['V'] == 0.0) and np.all(b0['F'] == 0.0)
    fr = dyn._run_raw(n, dt, *args, seed=seed, stride=1)
    hills = dyn._get_hills_raw()
    n_dep = mo.n_deposits(start, n, pace)
    assert list(hills[0]) == [NW * n_dep] * NG
    s = dyn.inv_mass.repeat(3)
    forces = _cuda_forces(gp)
    h, c1, sigma = mo.md_oracle.constants(dt, gamma, kT, s)
    worst = {}
    # Each step restated from the device's frame before it: CUDA's exp and atan2 may differ from NumPy's in the last
    # bit, which moves the bias force in its last bits and R, V and the CVs by about 1e-16 of their size per step (the
    # D = 36 fixture shows 1e-16 everywhere).  pbc_n6_m8's energy and forces are sums of terms of both signs (see
    # test_npt.py) whose cancellation turns such a last-bit change of R into about 1e-11 of E_pot and of the forces,
    # so of V and E_kin through the last half-kick; those and the bias are held to 1e-9.
    for f in range(n):
        c = start + f + 1
        Rp, Vp = (R0, V0) if f == 0 else (fr['R'][f - 1], fr['V'][f - 1])
        _, Fm = forces(Rp)
        _, _, Fb, touched = mo.bias(Rp, dyn.cvs, NW, _hills_before(hills, [0] * NG, c - 1, start, pace, NW))
        F = mo.total_force(Fm, Fb, touched)
        V = Vp + h * (F * s)
        R = Rp + h * V
        V = c1 * V + sigma * mo.md_oracle.normals(seed, c - 1, R.shape[0], R.shape[1])
        R = R + h * V
        E, Fm = forces(R)
        cv, Vb, Fb, touched = mo.bias(R, dyn.cvs, NW, _hills_before(hills, [0] * NG, c, start, pace, NW))
        V = V + h * (mo.total_force(Fm, Fb, touched) * s)
        for k, ref in (('R', R), ('V', V), ('E_pot', E), ('E_kin', mo.md_oracle.kinetic(V, s)), ('cv', cv),
                       ('bias', Vb)):
            e = rel_err(fr[k][f], ref)
            worst[k] = max(worst.get(k, 0.0), e)
            assert e < (1e-9 if k in ('V', 'E_pot', 'E_kin', 'bias') else 1e-11), (f, k, e)
        if c % pace == 0:  # the deposit: the state's CVs, the run's widths, w0 exp(-V / dkT) of the state's bias
            k = (c - 1) // pace - start // pace
            for g in range(NG):
                sl = slice(hills[0][:g].sum() + NW * k, hills[0][:g].sum() + NW * (k + 1))
                assert np.array_equal(hills[1][sl], fr['cv'][f][g * NW:(g + 1) * NW])
                assert np.all(hills[2][sl] == widths)
                assert rel_err(hills[3][sl], w0 * np.exp(-fr['bias'][f][g * NW:(g + 1) * NW] / dkT)) < 1e-15
    assert np.max(fr['bias'][-1]) > 0.1 * w0  # the bias is in play
    # The whole run restated from the start: the last-bit differences grow along the trajectory.  On n9_m16_s6 they
    # stay at 1.5e-14; pbc_n6_m8's cancellation (above) grows them to about 1.3e-7 over the 60 steps.
    fin, ref = mo.run(forces, R0, V0, s, dyn.cvs, NW, mo.empty_hills(NG, 4), n, dt, gamma, kT, w0, widths, pace, dkT,
                      seed=seed, step0=start, stride=1)
    whole = max(rel_err(fr[k], ref[k]) for k in ref)
    print('%s: worst per-step deviation %s, whole run %.3g' % (name, worst, whole))
    assert whole < (1e-6 if name == 'pbc_n6_m8' else 1e-12)
    assert [len(g[2]) for g in fin[6]] == list(hills[0])
    st = dyn._get_state_raw()
    assert np.array_equal(st['R'], fr['R'][-1]) and np.array_equal(st['E_pot'], fr['E_pot'][-1])
    assert np.array_equal(st['F'], forces(st['R'])[1])  # get_state's F is the model's
    b = dyn._get_bias_raw()
    assert np.array_equal(b['cv'], fr['cv'][-1]) and np.array_equal(b['V'], fr['bias'][-1])


def test_zero_height_is_md_run():
    import sgdml_b200

    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')
    gamma, kT, _, widths, pace, dkT = args
    md = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), n_replicas=NW * NG,
                                 E_to_eV=1.0, F_to_eV_Ang=1.0)
    dyn._set_state_raw(R0, V0, step=11)
    md._set_state_raw(R0, V0, step=11)
    a = dyn._run_raw(30, dt, gamma, kT, 0.0, widths, pace, dkT, seed=3, stride=10)
    b = md._run_raw(30, dt, gamma, kT, seed=3, stride=10)
    for k in ('R', 'V', 'E_pot', 'E_kin'):
        assert np.array_equal(a[k], b[k]), k
    assert np.all(a['bias'] == 0.0)
    assert _same(dyn._get_state_raw(), md._get_state_raw())
    n, _, _, H = dyn._get_hills_raw()
    assert list(n) == [NW * 10] * NG and np.all(H == 0.0)


def test_graph_matches_plain_launches_and_chunks(monkeypatch):
    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')

    def run(d):
        d._set_hills_raw([0] * NG, np.zeros((0, 4)), np.zeros((0, 4)), np.zeros(0))
        d._set_state_raw(R0, V0)
        out = d._run_raw(24, dt, *args, seed=8, stride=4)
        return out, d._get_hills_raw(), d._get_bias_raw()

    a = run(dyn)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = run(dyn)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    _, dc, _, _, _, _ = _setup('n9_m16_s6', chunk=2)
    c = run(dc)
    for x in (b, c):
        assert _same(a[0], x[0]) and all(np.array_equal(u, v) for u, v in zip(a[1], x[1])) and _same(a[2], x[2])


def test_continuation_and_restart_from_hills():
    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')
    _, dyn2, _, _, _, _ = _setup('n9_m16_s6')
    for d in (dyn, dyn2):
        d._set_state_raw(R0, V0, step=5)
    a = dyn._run_raw(40, dt, *args, seed=99, stride=5)
    b1 = dyn2._run_raw(20, dt, *args, seed=99, stride=5)
    b2 = dyn2._run_raw(20, dt, *args, seed=99, stride=5)
    assert _same(a, {k: np.concatenate([b1[k], b2[k]]) for k in a})
    ha = dyn._get_hills_raw()
    assert all(np.array_equal(u, v) for u, v in zip(ha, dyn2._get_hills_raw()))
    # restart: a fresh handle with the first half's state and hills continues bit for bit
    _, dyn3, _, _, _, _ = _setup('n9_m16_s6')
    dyn2._set_state_raw(R0, V0, step=5)
    dyn2._set_hills_raw([0] * NG, np.zeros((0, 4)), np.zeros((0, 4)), np.zeros(0))
    dyn2._run_raw(20, dt, *args, seed=99)
    st, hills = dyn2._get_state_raw(), dyn2._get_hills_raw()
    dyn3._set_state_raw(st['R'], st['V'], step=st['step'])  # V: the handle's half-step velocities
    dyn3._set_hills_raw(*hills)
    assert _same(dyn3._get_bias_raw(), dyn2._get_bias_raw())
    c2 = dyn3._run_raw(20, dt, *args, seed=99, stride=5)
    assert _same(b2, c2)
    assert all(np.array_equal(u, v) for u, v in zip(ha, dyn3._get_hills_raw()))


def test_isolated_from_predict_calls_and_other_handles():
    import torch

    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')
    _, ref, _, _, _, _ = _setup('n9_m16_s6')
    _, other, _, _, _, _ = _setup('n9_m16_s6', n_cv=2, nw=3, ng=2)
    out = []
    Rbig = np.tile(R0, (15, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((90, R0.shape[1]))
    for d, meddle in ((ref, False), (dyn, True)):
        d._set_state_raw(R0, V0)
        r1 = d._run_raw(12, dt, *args, seed=2, stride=4)
        if meddle:
            gp.predict(Rbig)
            gp.predict_hvp(Rbig, np.ones_like(Rbig))
            gp.predict(torch.from_numpy(Rbig).cuda())
            other._set_state_raw(R0[:6] + 0.01, V0[:6])
            other._run_raw(9, dt, args[0], args[1], 5 * args[2], args[3][:2], 1, np.inf, seed=2)
        r2 = d._run_raw(12, dt, *args, seed=2, stride=4)
        out.append((r1, r2, d._get_state_raw(), d._get_bias_raw()))
    assert all(_same(x, y) for x, y in zip(out[0], out[1]))
    assert all(np.array_equal(u, v) for u, v in zip(ref._get_hills_raw(), dyn._get_hills_raw()))


def test_handle_kind_rules_and_bad_input():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, dyn, R0, V0, dt, args = _setup('n9_m16_s6')
    L = _lib.lib()
    st = _lib.current_stream()
    masses = md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms))
    inv_mass = dyn.inv_mass
    h = ctypes.c_void_p()
    good_t, good_a = np.array([0, 2], dtype=np.int32), np.array([[0, 1, 0, 0], [0, 1, 2, 3]], dtype=np.int64)
    for t, a, n_cv in ((np.array([3, 0], dtype=np.int32), good_a, 2), (good_t, good_a * 0, 2),
                       (good_t, good_a + 6, 2), (good_t, good_a, 5), (good_t, good_a, 0)):
        assert L.sgdml_b200_metad_create(ctypes.byref(h), gp._handle, 2, 2, inv_mass.ctypes.data, n_cv,
                                         t.ctypes.data, a.ctypes.data) <= -1000 and not h.value
    with pytest.raises(_lib.EngineError):
        dyn._run_raw(10, dt, *args)  # no state yet
    with pytest.raises(_lib.EngineError):
        dyn._get_bias_raw()
    dyn._set_state_raw(R0, V0, step=7)
    dyn._run_raw(6, dt, *args, seed=1)
    H = dyn._handle
    # bad runs and hills change nothing (which handles metad_* take: tests/test_md_handle_kinds.py)
    before = dyn._get_state_raw(), dyn._get_bias_raw(), dyn._get_hills_raw()
    gamma, kT, w0, widths, pace, dkT = args
    good = dict(n_steps=6, dt=dt, gamma=gamma, kT=kT, w0=w0, widths=widths, pace=pace, dkT=dkT, stride=0)
    for bad in (dict(w0=-1.0), dict(w0=np.nan), dict(w0=np.inf), dict(widths=np.array([0.1, 0.0, 0.1, 0.1])),
                dict(widths=np.array([0.1, np.inf, 0.1, 0.1])), dict(pace=0), dict(dkT=0.0), dict(dkT=-np.inf),
                dict(dkT=np.nan), dict(gamma=np.nan), dict(stride=4), dict(dt=0.0), dict(n_steps=-1), dict(kT=-1.0)):
        kw = dict(good, **bad)
        out = {k: np.full((6, NW * NG, 27), 1.5) for k in ('R', 'cv')}
        wd = np.ascontiguousarray(kw['widths'], dtype=np.float64)
        rc = L.sgdml_b200_metad_run(H, kw['n_steps'], kw['dt'], kw['gamma'], kw['kT'], kw['w0'], wd.ctypes.data,
                                    kw['pace'], kw['dkT'], 0, kw['stride'], out['R'].ctypes.data, None, None, None,
                                    out['cv'].ctypes.data, None, st)
        assert rc <= -1000, bad
        assert np.all(out['R'] == 1.5) and np.all(out['cv'] == 1.5)
    one = np.array([1] + [0] * (NG - 1), dtype=np.int64)
    for c, wd, ht in ((np.zeros((1, 4)), np.zeros((1, 4)), np.ones(1)), (np.zeros((1, 4)), np.ones((1, 4)),
                                                                        np.full(1, np.nan)),
                      (np.full((1, 4), np.inf), np.ones((1, 4)), np.ones(1))):
        assert L.sgdml_b200_metad_set_hills(H, one.ctypes.data, c.ctypes.data, wd.ctypes.data, ht.ctypes.data,
                                            st) <= -1000
    assert L.sgdml_b200_metad_set_hills(H, (-one).ctypes.data, None, None, None, st) <= -1000
    after = dyn._get_state_raw(), dyn._get_bias_raw(), dyn._get_hills_raw()
    assert _same(before[0], after[0]) and _same(before[1], after[1])
    assert all(np.array_equal(u, v) for u, v in zip(before[2], after[2]))
    with pytest.raises(ValueError):
        sgdml_b200.GDMLMetadynamics(gp, masses, [('torsion', (0, 1, 2, 3))])
    with pytest.raises(ValueError):
        sgdml_b200.GDMLMetadynamics(gp, masses, [('angle', (0, 1))])
    pub = sgdml_b200.GDMLMetadynamics(gp, masses, [('distance', (0, 1))])
    pub.set_state(R0[0].reshape(-1, 3))
    with pytest.raises(ValueError):
        pub.run(5, 0.1, 300.0, 0.01, 0.01, [0.1], 2, bias_factor=1.0)


def test_public_units():
    """GDMLMetadynamics in eV / Angstrom / fs with a kcal/mol model against the raw calls in model units; torch in,
    torch out; the free energy from the hills."""
    import torch

    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc

    gp, raw, R0, V0, dt, args = _setup('n9_m16_s6')
    gamma, kT, w0, widths, pace, dkT = args
    masses = md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms))
    pub = sgdml_b200.GDMLMetadynamics(gp, masses * kc, CVS, n_walkers=NW, n_groups=NG)  # the same inverse masses
    assert np.allclose(pub.inv_mass, raw.inv_mass, rtol=1e-15)
    from sgdml_b200.md import KB_EV

    T = kT * kc / KB_EV
    bf = 1.0 + dkT / kT
    raw._set_state_raw(R0, V0)
    a = raw._run_raw(12, dt, gamma, kT, w0, widths, pace, dkT, seed=4, stride=4)
    pub.set_state(torch.from_numpy(R0.reshape(NG, NW, -1, 3)).cuda(), torch.from_numpy(V0).cuda().reshape(NG, NW, -1, 3))
    b = pub.run(12, dt, T, gamma, w0 * kc, widths, pace, bias_factor=bf, seed=4, stride=4)
    assert isinstance(b['cv'], torch.Tensor)
    assert rel_err(b['positions'].cpu().numpy().reshape(a['R'].shape), a['R']) < 1e-13
    assert rel_err(b['cv'].cpu().numpy().reshape(a['cv'].shape), a['cv']) < 1e-13
    assert rel_err(b['bias_energy'].cpu().numpy().ravel() / kc, a['bias'].ravel()) < 1e-12
    st = pub.get_state()
    rb = raw._get_bias_raw()
    assert st['cv'].shape == (NG, NW, 4) and st['bias_forces'].shape == (NG, NW, gp.n_atoms, 3)
    assert rel_err(st['bias_forces'].cpu().numpy().reshape(rb['F'].shape) / kc, rb['F']) < 1e-12
    hills = pub.hills()
    n, C, W, H = raw._get_hills_raw()
    assert len(hills) == NG and rel_err(np.concatenate([g['heights'] for g in hills]) / kc, H) < 1e-13
    # free energy on a grid of the first two CVs of a two-CV handle from the same hills
    two = sgdml_b200.GDMLMetadynamics(gp, masses * kc, CVS[:2], n_groups=2)
    two.set_hills([{'centers': [[1.0, 2.0]], 'widths': [[0.1, 0.2]], 'heights': [0.3]},
                   {'centers': np.zeros((0, 2)), 'widths': np.zeros((0, 2)), 'heights': np.zeros(0)}])
    fe = two.free_energy((np.array([1.0, 1.1]), np.array([2.0])), bias_factor=4.0)
    assert fe.shape == (2, 2, 1) and fe[0, 0, 0] == 0.0
    assert abs(fe[0, 1, 0] - 0.3 * (4 / 3) * (1 - np.exp(-0.5))) < 1e-12
    assert np.all(fe[1] == 0.0)


# ---------------------------------------------------------------------------------------------------- physics
def _dw_model():
    import sgdml_b200
    from test_neb import _dw_task

    return sgdml_b200.GDMLPredict(sgdml_b200.GDMLTrain().train(_dw_task()))


def _d01(R):
    X = np.asarray(R).reshape(-1, 4, 3)
    return np.linalg.norm(X[:, 0] - X[:, 1], axis=-1)


@pytest.fixture(scope='module')
def dw_model():
    return _dw_model()


def test_metadynamics_crosses_the_barrier_at_low_temperature(dw_model):
    """At kT = 0.006 (barrier 0.1), where test_remd.py shows plain Langevin stay in its well, metadynamics on d01
    visits both wells."""
    import sgdml_b200
    from test_neb import _DW_DC, _DW_PHI, _dw_hinge

    dyn = sgdml_b200.GDMLMetadynamics(dw_model, md_fs_masses(np.ones(4)), [('distance', (0, 1))], n_walkers=8,
                                      E_to_eV=1.0, F_to_eV_Ang=1.0)
    dyn._set_state_raw(np.tile(_dw_hinge(_DW_PHI[0]).reshape(1, 12), (8, 1)))
    fr = dyn._run_raw(10000, 0.02, 1.0, 0.006, 0.005, [0.05], 50, 10 * 0.006, seed=6, stride=10)
    d = fr['cv'][..., 0]
    print('metadynamics at kT 0.006: d01 in [%.3f, %.3f], barrier at %.3f, far well %.3f of the time'
          % (d.min(), d.max(), _DW_DC, (d > _DW_DC).mean()))
    assert (d < _DW_DC).any() and (d > _DW_DC).any()
    assert np.allclose(d, _d01(fr['R']).reshape(d.shape), rtol=0, atol=1e-12)


def test_well_tempered_profile_matches_unbiased_sampling(dw_model):
    """At kT = 0.04 (barrier 2.5 kT) unbiased Langevin of 64 replicas crosses often, and -kT ln of its d01 histogram is
    the free-energy profile.  Four independent groups of 8 well-tempered walkers (bias factor 6) each give
    -6/5 V(d01); the well-to-well free-energy difference and the barrier of their mean must agree with the histogram's
    within four standard errors of that mean across groups plus the histogram's own error (0.25 kT)."""
    import sgdml_b200
    from test_neb import _DW_DC, _DW_PHI, _dw_hinge

    kT, dt, gamma = 0.04, 0.02, 1.0
    masses = md_fs_masses(np.ones(4))
    A = _dw_hinge(_DW_PHI[0]).reshape(1, 12)
    B = _dw_hinge(_DW_PHI[1]).reshape(1, 12)
    md = sgdml_b200.GDMLDynamics(dw_model, masses, n_replicas=64, E_to_eV=1.0, F_to_eV_Ang=1.0)
    md._set_state_raw(np.concatenate([np.tile(A, (32, 1)), np.tile(B, (32, 1))]))
    md._run_raw(2000, dt, gamma, kT, seed=1)
    d_unb = _d01(md._run_raw(40000, dt, gamma, kT, seed=2, stride=20, frames=('R',))['R'])
    edges = np.linspace(np.quantile(d_unb, 0.002), np.quantile(d_unb, 0.998), 31)
    mid = 0.5 * (edges[1:] + edges[:-1])
    p, _ = np.histogram(d_unb, edges)
    F_unb = -kT * np.log(np.maximum(p, 1) / p.max())

    n_groups = 4
    dyn = sgdml_b200.GDMLMetadynamics(dw_model, masses, [('distance', (0, 1))], n_walkers=8, n_groups=n_groups,
                                      E_to_eV=1.0, F_to_eV_Ang=1.0)
    dyn._set_state_raw(np.tile(np.concatenate([np.tile(A, (4, 1)), np.tile(B, (4, 1))]), (n_groups, 1)))
    bf = 6.0
    dyn._run_raw(40000, dt, gamma, kT, 0.2 * kT, [0.04], 100, (bf - 1) * kT, seed=3)
    dyn.bias_factor = bf
    F_md = dyn.free_energy(mid) * 1.0  # (n_groups, bins), model units (E_to_eV = 1)

    def summary(F):
        left, right = mid < _DW_DC, mid > _DW_DC
        fl = -kT * np.log(np.exp(-F[left] / kT).sum())
        fr_ = -kT * np.log(np.exp(-F[right] / kT).sum())
        between = (mid > mid[left][np.argmin(F[left])]) & (mid < mid[right][np.argmin(F[right])])
        return fr_ - fl, F[between].max() - min(F[left].min(), F[right].min())

    ref = summary(F_unb)
    per = np.array([summary(f) for f in F_md])
    mean, sem = per.mean(0), per.std(0, ddof=1) / np.sqrt(n_groups)
    tol = 4.0 * sem + 0.25 * kT
    print('unbiased dF %.4f barrier %.4f; metadynamics dF %.4f +- %.4f, barrier %.4f +- %.4f (kT %.3f)'
          % (ref[0], ref[1], mean[0], sem[0], mean[1], sem[1], kT))
    assert np.all(np.abs(mean - np.array(ref)) < tol), (mean, ref, tol)
