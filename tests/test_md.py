"""Molecular dynamics on the device (sgdml_b200_md_*, sgdml_b200.GDMLDynamics) against the NumPy restatement of
tests/md_oracle.py.

CPU: Philox and its normals, the restatement's time reversibility on the oracle predictor, and the loud failure
without a device.  GPU: NVE and Langevin trajectories against the restatement driven by GDMLPredict.predict in every
predictor form, reproducibility and continuation, graph against plain launches, chunking, isolation from the
predictor's own calls, equipartition, energy conservation on a trained harmonic model, and argument errors.
"""

import ctypes
import os

import numpy as np
import pytest

import md_oracle
from conftest import rel_err
from md_common import FIXTURES_MD, _K_SPRING, _N_SPRING, _cuda_forces, md_fs_masses, spring_task  # noqa: F401


# ---------------------------------------------------------------------------------------------------- CPU
def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
              (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        got = md_oracle.philox4x32_10(np.array(ctr, dtype=np.uint64), key)
        assert tuple(int(x) for x in got) == want


def test_normals_moments():
    xi = md_oracle.normals(seed=(3 << 32) + 11, step=(1 << 32) + 5, n_rep=1000, dimi=1000).ravel()
    n = xi.size
    assert n == 10**6
    assert abs(xi.mean()) < 5.0 / np.sqrt(n)
    assert abs(xi.var() - 1.0) < 5.0 * np.sqrt(2.0 / n)
    # odd 3N drops the last sine; every other draw is unchanged
    assert np.array_equal(md_oracle.normals(1, 2, 3, 27), md_oracle.normals(1, 2, 3, 28)[:, :27])


def test_restated_verlet_is_time_reversible():
    from conftest import golden_model, load_golden
    from oracle import predict as opredict

    g = load_golden('n9_m16_s6')
    pred = opredict.Predictor(golden_model(g))
    R0 = np.asarray(g['R_query'], dtype=np.float64)[:2].reshape(2, -1)
    s = np.full(R0.shape[1], 0.05)
    E0, F0 = pred.predict(R0)
    dt = np.sqrt(2e-3 / np.max(np.abs(F0 * s)))
    V0 = np.random.default_rng(0).standard_normal(R0.shape) * 1e-3 / dt
    (R1, V1, _, _), _ = md_oracle.run(pred.predict, R0, V0, s, 50, dt)
    assert rel_err(R1, R0) > 1e-3  # it moved
    (R2, V2, _, _), _ = md_oracle.run(pred.predict, R1, -V1, s, 50, dt)
    assert np.max(np.abs(R2 - R0)) < 1e-10
    assert np.max(np.abs(-V2 - V0)) < 1e-10 * max(1.0, np.max(np.abs(V0)))


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_dynamics_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLDynamics({'type': 'm'}, np.ones(3))
    rc = _lib.lib().sgdml_b200_md_create(ctypes.byref(ctypes.c_void_p()), None, 1, np.ones(3).ctypes.data)
    assert rc == -1002  # SGDML_B200_ERR_NO_DEVICE


def test_md_entry_points_are_bound():
    from sgdml_b200 import _lib

    for name in ('create', 'destroy', 'set_state', 'get_state', 'run'):
        assert 'sgdml_b200_md_' + name in _lib.SIGNATURES


def test_ase_units():
    """The time unit and Boltzmann constant are ASE's (CODATA 2014): ase.units.fs and ase.units.kB."""
    from sgdml_b200 import md

    assert abs(md.FS - 0.09822694788464063) < 1e-16
    assert abs(md.KB_EV - 8.617330337217213e-05) < 1e-19


# ---------------------------------------------------------------------------------------------------- GPU helpers
def _setup(name, n_rep=3, chunk=0, slices=0):
    """(GDMLPredict, GDMLDynamics in model units (E_to_eV = F_to_eV_Ang = 1), R0, V0, dt)."""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    gp = sgdml_b200.GDMLPredict(model)
    if slices:
        gp.set_contraction_slices(slices)
    N = gp.n_atoms
    masses = md_fs_masses(np.linspace(1.0, 16.0, N))
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        dyn = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=n_rep, E_to_eV=1.0, F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    R0 = np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)
    R0 = R0[np.arange(n_rep) % R0.shape[0]].copy()
    if n_rep > Rq.shape[0]:
        R0 += 1e-3 * np.random.default_rng(1).standard_normal(R0.shape)
    _, F0 = gp.predict(R0)
    s = dyn.inv_mass.repeat(3)
    dt = float(np.sqrt(2e-3 / np.max(np.abs(F0 * s))))
    V0 = np.random.default_rng(2).standard_normal(R0.shape) * 1e-3 / dt
    return gp, dyn, R0, V0, dt


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in a) and set(a) == set(b)


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_nve_matches_host_loop(name):
    gp, dyn, R0, V0, dt = _setup(name)
    s = dyn.inv_mass.repeat(3)
    dyn._set_state_raw(R0, V0)
    fr = dyn._run_raw(20, dt, stride=5)
    forces = _cuda_forces(gp)
    (R, V, F, E), ref = md_oracle.run(forces, R0, V0, s, 20, dt, stride=5)
    print('%s: R bit-identical to the host loop: %s' % (name, np.array_equal(fr['R'], ref['R'])))
    assert rel_err(fr['R'], ref['R']) < 1e-12
    assert rel_err(fr['V'], ref['V']) < 1e-12
    for k in range(fr['R'].shape[0]):
        Ek, _ = gp.predict(fr['R'][k])
        assert rel_err(fr['E_pot'][k], Ek) < 1e-12
    assert rel_err(fr['E_kin'], md_oracle.kinetic(fr['V'], s)) < 1e-14
    assert rel_err(fr['E_kin'], ref['E_kin']) < 1e-11
    st = dyn._get_state_raw()
    assert st['step'] == 20
    assert np.array_equal(st['R'], fr['R'][-1]) and np.array_equal(st['V'], fr['V'][-1])
    assert rel_err(st['F'], F) < 1e-11


@pytest.mark.gpu
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_langevin_matches_host_loop(name):
    gp, dyn, R0, V0, dt = _setup(name)
    s = dyn.inv_mass.repeat(3)
    gamma = 0.1 / dt
    kT = float(np.mean(V0 * V0 / s))
    seed = (7 << 32) + 3
    dyn._set_state_raw(R0, V0, step=(1 << 32) - 10)  # the counter crosses 2^32 inside the run
    fr = dyn._run_raw(20, dt, gamma, kT, seed, stride=5)
    (R, V, _, _), ref = md_oracle.run(_cuda_forces(gp), R0, V0, s, 20, dt, gamma, kT, seed, step0=(1 << 32) - 10,
                                      stride=5)
    assert rel_err(fr['R'], ref['R']) < 1e-11
    assert rel_err(fr['V'], ref['V']) < 1e-11
    assert rel_err(fr['E_kin'], ref['E_kin']) < 1e-10


@pytest.mark.gpu
def test_int8_slices_and_slice_change():
    """D > 256 with the contractions on int8 slices, switched after the handle exists: the handle re-sizes its own
    workspace and follows the model."""
    gp, dyn, R0, V0, dt = _setup('big_n100_m2_s12')
    s = dyn.inv_mass.repeat(3)
    dyn._set_state_raw(R0, V0)
    dyn._run_raw(5, dt)
    gp.set_contraction_slices(6)
    dyn._set_state_raw(R0, V0)
    fr = dyn._run_raw(10, dt, stride=5)
    _, ref = md_oracle.run(_cuda_forces(gp), R0, V0, s, 10, dt, stride=5)
    assert rel_err(fr['R'], ref['R']) < 1e-12
    assert rel_err(fr['V'], ref['V']) < 1e-12


@pytest.mark.gpu
def test_reproducible_and_continuable():
    gp, dyn, R0, V0, dt = _setup('n9_m16_s6', n_rep=4)
    import sgdml_b200

    s = dyn.inv_mass.repeat(3)
    args = (0.05 / dt, float(np.mean(V0 * V0 / s)))
    dyn2 = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), n_replicas=4, E_to_eV=1.0,
                                   F_to_eV_Ang=1.0)
    dyn._set_state_raw(R0, V0, step=5)
    a = dyn._run_raw(40, dt, *args, seed=99, stride=5)
    sa = dyn._get_state_raw()
    dyn2._set_state_raw(R0, V0, step=5)
    b1 = dyn2._run_raw(20, dt, *args, seed=99, stride=5)
    b2 = dyn2._run_raw(20, dt, *args, seed=99, stride=5)
    sb = dyn2._get_state_raw()
    assert _same(a, {k: np.concatenate([b1[k], b2[k]]) for k in a})
    assert _same(sa, sb) and sa['step'] == 45
    dyn2._set_state_raw(R0, V0, step=5)
    assert _same(a, dyn2._run_raw(40, dt, *args, seed=99, stride=5))
    dyn2._set_state_raw(R0, V0, step=5)
    c = dyn2._run_raw(40, dt, *args, seed=100, stride=5)
    assert not np.array_equal(a['R'], c['R'])


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12', 'pbc_n6_m8'])
def test_graph_matches_plain_launches_and_chunks(name, monkeypatch):
    gp, dyn, R0, V0, dt = _setup(name, n_rep=5)
    s = dyn.inv_mass.repeat(3)
    args = (dt, 0.05 / dt, float(np.mean(V0 * V0 / s)), 4)
    dyn._set_state_raw(R0, V0)
    a = dyn._run_raw(20, *args, stride=5)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    dyn._set_state_raw(R0, V0)
    b = dyn._run_raw(20, *args, stride=5)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    _, dc, _, _, _ = _setup(name, n_rep=5, chunk=2)
    dc._set_state_raw(R0, V0)
    c = dc._run_raw(20, *args, stride=5)
    for k in a:
        assert rel_err(c[k], a[k]) < 1e-12, k


@pytest.mark.gpu
def test_isolated_from_predict_calls():
    import torch

    gp, dyn, R0, V0, dt = _setup('n12_m8_s12')
    import sgdml_b200

    masses = md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms))
    ref = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    ref._set_state_raw(R0, V0)
    a1 = ref._run_raw(10, dt, stride=5)
    a2 = ref._run_raw(10, dt, stride=5)
    sa = ref._get_state_raw()

    Rbig = np.tile(R0, (30, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((90, R0.shape[1]))
    E_before, F_before = gp.predict(R0)
    Eb_before, Fb_before = gp.predict(Rbig)
    dyn._set_state_raw(R0, V0)
    b1 = dyn._run_raw(10, dt, stride=5)
    gp.predict(Rbig)
    gp.predict_hvp(Rbig, np.ones_like(Rbig))
    gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (90, 1, 1)))
    b2 = dyn._run_raw(10, dt, stride=5)
    assert _same(a1, b1) and _same(a2, b2) and _same(sa, dyn._get_state_raw())
    E_after, F_after = gp.predict(R0)
    Eb_after, Fb_after = gp.predict(Rbig)
    assert np.array_equal(E_before, E_after) and np.array_equal(F_before, F_after)
    assert np.array_equal(Eb_before, Eb_after) and np.array_equal(Fb_before, Fb_after)


@pytest.mark.gpu
def test_equipartition():
    """<E_kin> over 256 replicas and 1000 steps is (3N / 2) kT within 5 standard errors (block averages of the
    run's own series; the seed is fixed)."""
    gp, dyn, R0, V0, dt = _setup('n9_m16_s6', n_rep=256)
    s = dyn.inv_mass.repeat(3)
    # kT well above the energy the synthetic model releases while the replicas relax from the query geometries, a step
    # short against the thermal motion (the O(dt^2) bias of the full-step velocities) and strong coupling
    kT = 30.0 * float(np.mean(V0 * V0 / s))
    dt = 0.5 * dt
    gamma = 0.5 / dt
    dyn._set_state_raw(R0, V0)
    dyn._run_raw(2000, dt, gamma, kT, seed=2024)
    fr = dyn._run_raw(1000, dt, gamma, kT, seed=2024, stride=10, frames=('E_kin',))
    series = fr['E_kin'].mean(1)  # (100,) replica means
    blocks = series.reshape(10, 10).mean(1)
    se = blocks.std(ddof=1) / np.sqrt(len(blocks))
    want = 1.5 * gp.n_atoms * kT
    print('<E_kin> = %.6g, (3N/2) kT = %.6g, standard error %.3g' % (series.mean(), want, se))
    assert abs(series.mean() - want) < 5.0 * se


# max |E_tot(t) - E_tot(0)| / E_kin(0) over 2000 velocity-Verlet steps (dt = 0.02 / omega of the stiffest spring) of
# the restatement (tests/md_oracle.run) on oracle.predict.Predictor trained on `spring_task`: 4.2e-5.  The bound leaves a
# factor of about 10 for the engine's own training of the same task.
_SPRING_DRIFT_BOUND = 4e-4


def _spring_setup():
    """R0, V0 (1, 3N), s (3N,) and dt of the conservation run."""
    from sgdml_b200 import synth

    R0 = synth.base_geometry(_N_SPRING).reshape(1, -1)
    s = np.full(3 * _N_SPRING, 0.1)
    omega = np.sqrt(4.0 * _K_SPRING * 0.1)
    dt = 0.02 / omega
    V0 = np.random.default_rng(11).standard_normal((_N_SPRING, 3)) * 0.03 * omega
    V0 = (V0 - V0.mean(0)).reshape(1, -1)  # no drift of the centre of mass (equal masses)
    return R0, V0, s, dt


def spring_drift(E_pot, E_kin, E_kin0):
    tot = E_pot + E_kin
    return float(np.max(np.abs(tot - tot[0])) / E_kin0)


@pytest.mark.gpu
def test_energy_conservation(spring_task):
    import sgdml_b200

    model = sgdml_b200.GDMLTrain().train(spring_task)
    gp = sgdml_b200.GDMLPredict(model)
    R0, V0, s, dt = _spring_setup()
    dyn = sgdml_b200.GDMLDynamics(gp, md_fs_masses(1.0 / s[::3]), E_to_eV=1.0, F_to_eV_Ang=1.0)
    assert np.allclose(dyn.inv_mass.repeat(3), s, rtol=1e-14)
    dyn._set_state_raw(R0, V0)
    fr = dyn._run_raw(2000, dt, stride=1, frames=('E_pot', 'E_kin'))
    E_kin0 = float(md_oracle.kinetic(V0, dyn.inv_mass.repeat(3))[0])
    drift = spring_drift(fr['E_pot'][:, 0], fr['E_kin'][:, 0], E_kin0)
    print('energy drift over 2000 steps: %.3g of E_kin(0)' % drift)
    assert drift < _SPRING_DRIFT_BOUND


@pytest.mark.gpu
def test_public_units():
    """GDMLDynamics in eV / Angstrom / fs against its model-unit form, with kcal/mol models (the default units)."""
    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc
    import hvp_oracle

    model, Rq, _ = hvp_oracle.fixture_model('n9_m16_s6')
    masses = np.linspace(1.0, 16.0, 9)
    d = sgdml_b200.GDMLDynamics(model, masses, n_replicas=2)
    R0 = np.asarray(Rq[:2], dtype=np.float64).reshape(2, 9, 3)
    V0 = 1e-3 * np.random.default_rng(0).standard_normal(R0.shape)
    d.set_state(R0, V0)
    out = d.run(10, 0.5, temperature_K=300.0, friction_per_fs=0.01, seed=1, stride=5)
    raw = sgdml_b200.GDMLDynamics(d.gdml_predict, masses, n_replicas=2)
    raw._set_state_raw(R0.reshape(2, -1), V0.reshape(2, -1))
    from sgdml_b200 import md

    f = raw._run_raw(10, 0.5, 0.01, md.KB_EV * 300.0 / kc, 1, 5)
    assert np.array_equal(out['positions'], f['R'].reshape(2, 2, 9, 3))
    assert np.allclose(out['potential_energy'], f['E_pot'] * kc, rtol=1e-15)
    assert np.allclose(out['kinetic_energy'], f['E_kin'] * kc, rtol=1e-15)
    st = d.get_state()
    assert st['step'] == 10 and st['positions'].shape == (2, 9, 3) and st['forces'].shape == (2, 9, 3)
    # CUDA tensors in -> CUDA tensors out
    import torch

    d.set_state(torch.from_numpy(R0).cuda(), torch.from_numpy(V0).cuda())
    t = d.run(10, 0.5, temperature_K=300.0, friction_per_fs=0.01, seed=1, stride=5)
    assert t['positions'].is_cuda and np.array_equal(t['positions'].cpu().numpy(), out['positions'])


@pytest.mark.gpu
def test_bad_input_is_rejected():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, dyn, R0, V0, dt = _setup('n9_m16_s6')
    L = _lib.lib()
    h = ctypes.c_void_p()
    assert L.sgdml_b200_md_create(ctypes.byref(h), None, 3, np.ones(9).ctypes.data) <= -1000 and not h.value
    with pytest.raises(_lib.EngineError):
        sgdml_b200.GDMLDynamics(gp, np.full(9, np.nan))
    with pytest.raises(_lib.EngineError):
        sgdml_b200.GDMLDynamics(gp, -np.ones(9))
    with pytest.raises(ValueError):
        sgdml_b200.GDMLDynamics(gp, np.ones(8))
    with pytest.raises(_lib.EngineError):
        dyn._run_raw(10, dt)  # no state yet
    with pytest.raises(ValueError):
        dyn._set_state_raw(R0[:2], V0[:2])
    dyn._set_state_raw(R0, V0, step=7)
    before = dyn._get_state_raw()
    for kw in (dict(n_steps=10, dt=dt, stride=3), dict(n_steps=10, dt=dt, kT=1.0), dict(n_steps=10, dt=0.0),
               dict(n_steps=10, dt=np.nan), dict(n_steps=10, dt=dt, gamma=-1.0), dict(n_steps=-1, dt=dt),
               dict(n_steps=10, dt=dt, gamma=1.0, kT=-1.0)):
        out = {k: np.full((4, 3, 27), 1.5) for k in ('R', 'V')}
        rc = L.sgdml_b200_md_run(dyn._handle, kw['n_steps'], kw['dt'], kw.get('gamma', 0.0), kw.get('kT', 0.0), 0,
                                 kw.get('stride', 0), out['R'].ctypes.data, out['V'].ctypes.data, None, None,
                                 _lib.current_stream())
        assert rc <= -1000, kw
        assert np.all(out['R'] == 1.5) and np.all(out['V'] == 1.5)
    assert _same(before, dyn._get_state_raw())
