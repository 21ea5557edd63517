"""Replica-exchange molecular dynamics on the device (sgdml_b200_remd_run, sgdml_b200.GDMLReplicaExchange) against the
NumPy restatement of tests/remd_oracle.py.

CPU: the schedule and pairing, no exchange at a run's first state and continuation, the acceptance frequency of the
exchange draw, its stream apart from the O noise, the reduction to md_oracle without exchanges, and the velocity rule.
GPU: the device against the restatement driven by GDMLPredict.predict in every predictor form, the reduction to
sgdml_b200_md_run, all-accepted swaps at equal temperatures, reproducibility and continuation, graph against plain
launches, chunks that split a ladder, isolation, MD and relaxation on the same handle afterwards, public units, argument
errors, the canonical ensemble at every slot, and barrier crossing on a trained double-well model that plain Langevin
at the same temperature does not achieve.
"""

import os

import numpy as np
import pytest

import md_oracle
import remd_oracle
from conftest import rel_err
from md_common import FIXTURES_MD, _cuda_forces, _spring_pes, md_fs_masses, spring_task  # noqa: F401


def _spring_forces(R):
    E, F = _spring_pes(R)
    return E, F.reshape(len(E), -1)


def _spring_state(n_rep, seed=0):
    from sgdml_b200 import synth

    rng = np.random.default_rng(seed)
    R0 = np.tile(synth.base_geometry(5).reshape(1, -1), (n_rep, 1)) + 0.05 * rng.standard_normal((n_rep, 15))
    V0 = 0.05 * rng.standard_normal((n_rep, 15))
    return R0, V0, np.full(15, 0.1)


# ---------------------------------------------------------------------------------------------------- CPU
def test_pairs_and_parity():
    assert remd_oracle.pairs(1, 1, 4) == [1] and remd_oracle.pairs(2, 1, 4) == [0, 2]
    assert remd_oracle.pairs(2, 1, 5) == [0, 2] and remd_oracle.pairs(3, 1, 5) == [1, 3]
    assert remd_oracle.pairs(3, 3, 4) == [1] and remd_oracle.pairs(6, 3, 4) == [0, 2]
    assert remd_oracle.pairs(9, 3, 4) == [1]
    assert remd_oracle.pairs(1, 1, 2) == [] and remd_oracle.pairs(2, 1, 2) == [0]
    for n_temps in range(2, 12):
        for c in range(1, 20):
            p = remd_oracle.pairs(c, 1, n_temps)
            assert all(k % 2 == c % 2 and k + 1 < n_temps for k in p)  # disjoint pairs of one parity
            assert len(p) == (n_temps - c % 2) // 2  # the kernel's count
    assert not remd_oracle.is_exchange(6, 6, 3)  # never on a run's first state
    assert remd_oracle.is_exchange(9, 6, 3) and not remd_oracle.is_exchange(8, 6, 3)
    assert not any(remd_oracle.is_exchange(c, 0, 0) for c in range(1, 10))  # every = 0: never


def test_no_exchange_at_run_start_and_continuation():
    R0, V0, s = _spring_state(6)
    kT = [0.02, 0.05, 0.1]
    args = (s, kT, 0.05, 0.5, 1)
    # one step from step index 6: only the state at 7 is exchanged (the pair (1, 2) of each ladder)
    _, _, one = remd_oracle.run(_spring_forces, R0, V0, *args[:2], 1, *args[2:], seed=3, step0=6)
    assert one['n_attempted'].tolist() == [[0, 1], [0, 1]]
    a_st, a_fr, a = remd_oracle.run(_spring_forces, R0, V0, *args[:2], 40, *args[2:], seed=3, step0=6, stride=5)
    b_st, b_fr, b = remd_oracle.run(_spring_forces, R0, V0, *args[:2], 20, *args[2:], seed=3, step0=6, stride=5)
    c_st, c_fr, c = remd_oracle.run(_spring_forces, b_st['R'], b_st['V'], *args[:2], 20, *args[2:], seed=3, step0=26,
                                    stride=5, F=b_st['F'], E=b_st['E'], walker=b_st['walker'])
    for k in a_st:
        assert np.array_equal(a_st[k], c_st[k]), k
    for k in a_fr:
        assert np.array_equal(a_fr[k], np.concatenate([b_fr[k], c_fr[k]])), k
    for k in ('n_accepted', 'n_attempted'):
        assert np.array_equal(a[k], b[k] + c[k])
    assert a['n_attempted'].sum() == 2 * 40 and 0 < a['n_accepted'].sum() < a['n_attempted'].sum()


def test_acceptance_frequency():
    """Over many draws at fixed energies the swap is accepted with probability min(1, exp(D)), within 5 standard
    errors."""
    beta = 1.0 / np.array([0.5, 1.0])
    c = np.arange(1, 200001, dtype=np.uint64)
    for dE in (0.05, 0.5, 1.0, 3.0, -0.4):
        d = remd_oracle.delta(beta, 0, -dE, 0.0)  # E_0 - E_1 = -dE, D = -dE (beta_0 - beta_1)
        u = remd_oracle.exchange_uniform(12345, 0, 3, c)
        acc = (d >= 0.0) | (u < np.exp(d))
        p = min(1.0, np.exp(d))
        se = np.sqrt(max(p * (1.0 - p), 1e-12) / len(c))
        assert abs(acc.mean() - p) < 5.0 * se + 1e-12, (dE, acc.mean(), p)


def test_exchange_stream_is_apart_from_the_noise():
    """The exchange counter's first word has the high bit set; the O noise's is a pair index below 2^31.  The same
    (k, l, c) without the bit gives another draw."""
    assert remd_oracle.EXCHANGE_BIT == 1 << 31
    k, l, c = np.meshgrid(np.arange(8), np.arange(4), np.arange(1, 50), indexing='ij')
    u = remd_oracle.exchange_uniform(77, k, l, c)
    ctr = np.stack([k, l, c, np.zeros_like(c)], axis=-1).astype(np.uint64)
    w = md_oracle.philox4x32_10(ctr, (77, 0))
    u_noise = md_oracle._uniform53(w[..., 0], w[..., 1])  # the U_a of coordinate pair k, replica l, step c
    assert not np.any(u == u_noise)
    assert len(np.unique(u)) == u.size


def test_without_exchanges_at_one_temperature_is_md():
    R0, V0, s = _spring_state(6)
    st, fr, stats = remd_oracle.run(_spring_forces, R0, V0, s, [0.05, 0.05, 0.05], 30, 0.05, 0.5, 0, seed=9, step0=4,
                                    stride=5)
    (R, V, F, E), ref = md_oracle.run(_spring_forces, R0, V0, s, 30, 0.05, 0.5, 0.05, seed=9, step0=4, stride=5)
    assert np.array_equal(st['R'], R) and np.array_equal(st['V'], V) and np.array_equal(st['E'], E)
    for k in ref:
        assert np.array_equal(fr[k], ref[k]), k
    assert np.all(fr['walker'] == np.arange(6)) and stats['n_attempted'].sum() == 0


def test_accepted_swap_rescales_the_velocity():
    """An accepted swap multiplies each configuration's full-step velocity by sqrt(kT_new / kT_old), to within one
    rounding (the device's v' = lam w - h F s, completed by the pending half-kick)."""
    R0, V0, s = _spring_state(2, seed=4)
    E, F = _spring_forces(R0)
    kT = [0.03, 0.12]
    st = {'R': R0.copy(), 'V': V0.copy(), 'F': F.copy(), 'E': np.array([1.0, 0.5]), 'walker': np.arange(2)}
    stats = {'n_accepted': np.zeros((1, 1), dtype=np.int64), 'n_attempted': np.zeros((1, 1), dtype=np.int64),
             'margin': np.inf}
    remd_oracle.exchange(st, 2, 1, 0, kT, 0.025, s, stats)  # D = (beta_0 - beta_1)(E_0 - E_1) > 0: accepted
    assert stats['n_accepted'][0, 0] == 1 and st['walker'].tolist() == [1, 0]
    assert np.array_equal(st['R'], R0[::-1]) and np.array_equal(st['F'], F[::-1]) and st['E'].tolist() == [0.5, 1.0]
    for slot, src, lam in ((0, 1, 0.5), (1, 0, 2.0)):
        want = lam * V0[src]
        kick = 0.025 * (F[src] * s)
        assert np.all(np.abs(st['V'][slot] - want) <= np.spacing(np.maximum(np.abs(want), np.abs(kick)))), slot


def test_entry_point_is_bound():
    from sgdml_b200 import _lib

    assert 'sgdml_b200_remd_run' in _lib.SIGNATURES


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLReplicaExchange({'type': 'm'}, np.ones(3), [300.0, 400.0])


# ---------------------------------------------------------------------------------------------------- GPU helpers
def _setup(name, n_ladders=2, n_temps=3, chunk=0, slices=0):
    """(GDMLPredict, GDMLReplicaExchange in model units, R0, V0, dt, kT): kT a ladder doubling per slot, its lowest
    temperature set by the spread of the starting energies so that the Metropolis test both accepts and rejects."""
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
        rex = sgdml_b200.GDMLReplicaExchange(gp, masses, np.ones(n_temps), n_ladders=n_ladders, E_to_eV=1.0,
                                             F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    n_rep = n_ladders * n_temps
    R0 = np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)
    R0 = R0[np.arange(n_rep) % R0.shape[0]].copy()
    R0 += 1e-3 * np.random.default_rng(1).standard_normal(R0.shape)
    E0, F0 = gp.predict(R0)
    s = rex.inv_mass.repeat(3)
    dt = float(np.sqrt(2e-3 / np.max(np.abs(F0 * s))))
    V0 = np.random.default_rng(2).standard_normal(R0.shape) * 1e-3 / dt
    kT = max(float(np.std(E0)), 1e-3 * float(np.max(np.abs(E0)))) * 2.0 ** np.arange(n_temps)
    return gp, rex, R0, V0, dt, kT


def _device(rex, R0, V0, n_steps, dt, gamma, kT, every, seed, stride=5, step=0):
    rex._set_state_raw(R0, V0, step=step)
    return rex._run_raw(n_steps, dt, gamma, kT, every, seed, stride)


def _same(a, b):
    return set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)


# ---------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_matches_restatement(name):
    gp, rex, R0, V0, dt, kT = _setup(name)
    s = rex.inv_mass.repeat(3)
    gamma, seed, step = 0.1 / dt, (5 << 32) + 21, (1 << 32) - 9  # the counter crosses 2^32 inside the run
    dev = _device(rex, R0, V0, 20, dt, gamma, kT, 2, seed, step=step)
    st, ref, stats = remd_oracle.run(_cuda_forces(gp), R0, V0, s, kT, 20, dt, gamma, 2, seed, step0=step, stride=5)
    print('%s: R bit-identical %s, accepted %s of %s, margin %.3g' % (
        name, np.array_equal(dev['R'], ref['R']), dev['n_accepted'].tolist(), dev['n_attempted'].tolist(),
        stats['margin']))
    assert stats['margin'] > 1e-9
    assert rel_err(dev['R'], ref['R']) < 1e-11
    assert rel_err(dev['V'], ref['V']) < 1e-11
    for k in range(dev['R'].shape[0]):  # each frame's E_pot is the model's at that frame's positions, as in test_md.py
        assert rel_err(dev['E_pot'][k], gp.predict(dev['R'][k])[0]) < 1e-12
    assert rel_err(dev['E_kin'], md_oracle.kinetic(dev['V'], s)) < 1e-14
    assert rel_err(dev['E_kin'], ref['E_kin']) < 1e-10
    assert np.array_equal(dev['walker'], ref['walker'])
    assert np.array_equal(dev['walkers'], st['walker'])
    assert np.array_equal(dev['n_accepted'], stats['n_accepted'])
    assert np.array_equal(dev['n_attempted'], stats['n_attempted'])
    assert stats['n_attempted'].sum() == 2 * 10  # 2 ladders, one pair per exchange of 3 slots, 10 exchanges
    raw = rex._get_state_raw()
    assert raw['step'] == step + 20 and np.array_equal(raw['R'], dev['R'][-1])


@pytest.mark.gpu
def test_int8_slices():
    gp, rex, R0, V0, dt, kT = _setup('big_n100_m2_s12', slices=6)
    s = rex.inv_mass.repeat(3)
    dev = _device(rex, R0, V0, 10, dt, 0.1 / dt, kT, 1, 3)
    st, ref, stats = remd_oracle.run(_cuda_forces(gp), R0, V0, s, kT, 10, dt, 0.1 / dt, 1, 3, stride=5)
    assert stats['margin'] > 1e-9
    assert rel_err(dev['R'], ref['R']) < 1e-11 and np.array_equal(dev['walker'], ref['walker'])


@pytest.mark.gpu
def test_one_temperature_without_exchanges_is_md_run():
    import sgdml_b200

    gp, rex, R0, V0, dt, kT = _setup('n9_m16_s6', n_ladders=2, n_temps=4)
    kT1 = float(kT[1])
    md = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), n_replicas=8, E_to_eV=1.0,
                                 F_to_eV_Ang=1.0)
    md._set_state_raw(R0, V0, step=3)
    want = md._run_raw(20, dt, 0.1 / dt, kT1, 11, 5)
    got = _device(rex, R0, V0, 20, dt, 0.1 / dt, np.full(4, kT1), 0, 11, step=3)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
    assert np.all(got['walker'] == np.arange(8)) and np.all(got['n_attempted'] == 0)
    a, b = rex._get_state_raw(), md._get_state_raw()
    assert _same(a, b)


@pytest.mark.gpu
def test_one_temperature_accepts_every_swap():
    gp, rex, R0, V0, dt, kT = _setup('n12_m8_s12', n_ladders=2, n_temps=4)
    got = _device(rex, R0, V0, 12, dt, 0.1 / dt, np.full(4, float(kT[0])), 1, 5, stride=1)
    assert np.array_equal(got['n_accepted'], got['n_attempted'])
    assert got['n_attempted'].tolist() == [[6, 6, 6]] * 2
    w = np.arange(8)
    for c in range(1, 13):
        for k in remd_oracle.pairs(c, 1, 4):
            for l in range(2):
                w[[4 * l + k, 4 * l + k + 1]] = w[[4 * l + k + 1, 4 * l + k]]
        assert np.array_equal(got['walker'][c - 1], w), c
    assert np.array_equal(got['walkers'], w)


@pytest.mark.gpu
def test_reproducible_and_continuable():
    gp, rex, R0, V0, dt, kT = _setup('n9_m16_s6', n_ladders=2, n_temps=4)
    a = _device(rex, R0, V0, 40, dt, 0.1 / dt, kT, 1, 99, step=5)
    sa = rex._get_state_raw()
    b1 = _device(rex, R0, V0, 20, dt, 0.1 / dt, kT, 1, 99, step=5)
    b2 = rex._run_raw(20, dt, 0.1 / dt, kT, 1, 99, 5)
    sb = rex._get_state_raw()
    for k in ('R', 'V', 'E_pot', 'E_kin', 'walker'):
        assert np.array_equal(a[k], np.concatenate([b1[k], b2[k]])), k
    for k in ('n_accepted', 'n_attempted'):
        assert np.array_equal(a[k], b1[k] + b2[k]), k
    assert np.array_equal(a['walkers'], b2['walkers'])
    assert _same(sa, sb) and sa['step'] == 45
    assert 0 < a['n_accepted'].sum() < a['n_attempted'].sum()
    assert _same(a, _device(rex, R0, V0, 40, dt, 0.1 / dt, kT, 1, 99, step=5))
    c = _device(rex, R0, V0, 40, dt, 0.1 / dt, kT, 1, 100, step=5)
    assert not np.array_equal(a['R'], c['R'])


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12', 'pbc_n6_m8'])
def test_graph_matches_plain_launches_and_chunks(name, monkeypatch):
    gp, rex, R0, V0, dt, kT = _setup(name)
    args = (R0, V0, 20, dt, 0.1 / dt, kT, 2, 4)
    a = _device(rex, *args)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _device(rex, *args)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    _, rc, _, _, _, _ = _setup(name, chunk=2)  # chunks of 2 geometries split the ladders of 3
    c = _device(rc, *args)
    for k in ('R', 'V', 'E_pot', 'E_kin'):
        assert rel_err(c[k], a[k]) < 1e-12, k
    for k in ('walker', 'walkers', 'n_accepted', 'n_attempted'):
        assert np.array_equal(c[k], a[k]), k


@pytest.mark.gpu
def test_isolated_from_predict_calls_and_other_handles():
    import torch

    import sgdml_b200

    gp, rex, R0, V0, dt, kT = _setup('n12_m8_s12')
    args = (dt, 0.1 / dt, kT, 1, 8, 5)
    masses = md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms))
    ref = sgdml_b200.GDMLReplicaExchange(gp, masses, np.ones(3), n_ladders=2, E_to_eV=1.0, F_to_eV_Ang=1.0)
    ref._set_state_raw(R0, V0)
    a1 = ref._run_raw(10, *args)
    a2 = ref._run_raw(10, *args)
    sa = ref._get_state_raw()

    other = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.ones(gp.n_atoms)), n_replicas=6, E_to_eV=1.0, F_to_eV_Ang=1.0)
    other._set_state_raw(R0)
    Rbig = np.tile(R0, (15, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((90, R0.shape[1]))
    E_before, F_before = gp.predict(Rbig)
    rex._set_state_raw(R0, V0)
    b1 = rex._run_raw(10, *args)
    gp.predict(Rbig)
    gp.predict_hvp(Rbig, np.ones_like(Rbig))
    other._run_raw(7, dt, 0.1 / dt, float(kT[0]), 3)
    gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (90, 1, 1)))
    b2 = rex._run_raw(10, *args)
    assert _same(a1, b1) and _same(a2, b2) and _same(sa, rex._get_state_raw())
    E_after, F_after = gp.predict(Rbig)
    assert np.array_equal(E_before, E_after) and np.array_equal(F_before, F_after)


@pytest.mark.gpu
def test_md_and_relaxation_on_the_same_handle_afterwards():
    """After replica-exchange runs (which grow the handle's noise table and capture their own step), the same handle
    runs Langevin MD and FIRE as test_md.py and test_relax.py expect, and replica exchange again."""
    import relax_oracle

    import sgdml_b200

    gp, rex, R0, V0, dt, kT = _setup('n9_m16_s6', n_ladders=1, n_temps=3)
    s = rex.inv_mass.repeat(3)
    first = _device(rex, R0, V0, 10, dt, 0.1 / dt, kT, 1, 4)
    gamma, kT1, seed = 0.1 / dt, float(kT[2]), (7 << 32) + 3
    rex._set_state_raw(R0, V0, step=(1 << 32) - 10)
    fr = sgdml_b200.GDMLDynamics._run_raw(rex, 20, dt, gamma, kT1, seed, stride=5)
    _, ref = md_oracle.run(_cuda_forces(gp), R0, V0, s, 20, dt, gamma, kT1, seed, step0=(1 << 32) - 10, stride=5)
    assert rel_err(fr['R'], ref['R']) < 1e-11
    assert rel_err(fr['V'], ref['V']) < 1e-11
    assert rel_err(fr['E_kin'], ref['E_kin']) < 1e-10
    rex._set_state_raw(R0)
    n, c, fm = sgdml_b200.GDMLRelaxation._relax_raw(rex, 'fire', 10, 0.0, 0.05, 0.5 * dt, 5.0 * dt)
    want = relax_oracle.fire(_cuda_forces(gp), R0, 10, 0.0, 0.05, 0.5 * dt, 5.0 * dt)
    assert rel_err(rex._get_state_raw()['R'], want['R']) < 1e-12 and np.all(n == 10)
    assert _same(first, _device(rex, R0, V0, 10, dt, 0.1 / dt, kT, 1, 4))


@pytest.mark.gpu
def test_public_units():
    """GDMLReplicaExchange in eV / Angstrom / fs / K (a kcal/mol model, the default units) against its model-unit form,
    broadcast starting geometries, and CUDA tensors in and out."""
    import torch

    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import md
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc

    model, Rq, _ = hvp_oracle.fixture_model('n9_m16_s6')
    masses = np.linspace(1.0, 16.0, 9)
    T = np.geomspace(300.0, 600.0, 3)
    rex = sgdml_b200.GDMLReplicaExchange(model, masses, T, n_ladders=2)
    R0 = np.asarray(Rq[:2], dtype=np.float64).reshape(2, 9, 3)
    V0 = 1e-3 * np.random.default_rng(0).standard_normal((2, 3, 9, 3))
    rex.set_state(R0, V0)  # (n_ladders, N, 3) positions go to every slot of their ladder
    out = rex.run(10, 0.5, 0.01, 2, seed=1, stride=5)
    raw = sgdml_b200.GDMLReplicaExchange(rex.gdml_predict, masses, T, n_ladders=2)
    raw._set_state_raw(np.repeat(R0, 3, 0).reshape(6, -1), V0.reshape(6, -1))
    f = raw._run_raw(10, 0.5, 0.01, md.KB_EV * T / kc, 2, 1, 5)
    assert np.array_equal(out['positions'], f['R'].reshape(2, 2, 3, 9, 3))
    assert np.allclose(out['velocities'], f['V'].reshape(2, 2, 3, 9, 3), rtol=1e-15, atol=0.0)
    assert np.allclose(out['potential_energy'], f['E_pot'].reshape(2, 2, 3) * kc, rtol=1e-15)
    assert np.allclose(out['kinetic_energy'], f['E_kin'].reshape(2, 2, 3) * kc, rtol=1e-15)
    assert np.array_equal(out['walker'], f['walker'].reshape(2, 2, 3)) and out['walker'].dtype == np.int32
    assert np.array_equal(out['walkers'], f['walkers'].reshape(2, 3))
    assert np.array_equal(out['n_accepted'], f['n_accepted']) and out['n_attempted'].dtype == np.int64
    att = out['n_attempted']
    assert np.array_equal(np.isnan(out['acceptance']), att == 0)
    assert np.allclose(out['acceptance'][att > 0], (out['n_accepted'] / np.maximum(att, 1))[att > 0])
    st = rex.get_state()
    assert st['step'] == 10 and st['positions'].shape == (2, 3, 9, 3) and st['potential_energy'].shape == (2, 3)
    assert rex.run(4, 0.5, 0.01, 1)['walkers'].shape == (2, 3)  # stride 0: no frames, the labels and counts
    # CUDA tensors in -> CUDA tensors out
    rex.set_state(torch.from_numpy(R0).cuda(), torch.from_numpy(V0).cuda())
    t = rex.run(10, 0.5, 0.01, 2, seed=1, stride=5)
    assert t['positions'].is_cuda and t['walker'].is_cuda and t['acceptance'].is_cuda
    assert np.array_equal(t['positions'].cpu().numpy(), out['positions'])
    assert np.array_equal(t['walkers'].cpu().numpy(), out['walkers'])
    one = sgdml_b200.GDMLReplicaExchange(rex.gdml_predict, masses, T)
    one.set_state(R0[0])  # (N, 3) goes to every slot
    assert one.get_state()['positions'].shape == (1, 3, 9, 3)
    with pytest.raises(ValueError):
        one.set_state(np.zeros((2, 2, 9, 3)))
    with pytest.raises(ValueError):
        sgdml_b200.GDMLReplicaExchange(rex.gdml_predict, masses, [300.0])


@pytest.mark.gpu
def test_bad_input_is_rejected():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, rex, R0, V0, dt, kT = _setup('n9_m16_s6')
    L = _lib.lib()
    h = rex._handle

    def call(handle, n_temps=3, kT=kT, n_steps=10, dt=dt, gamma=1.0, every=1, stride=5):
        kT = np.ascontiguousarray(kT, dtype=np.float64)
        out = [np.full((2, 6, 27), 1.5) for _ in range(2)] + [np.full((2, 6), 1.5) for _ in range(2)]
        out += [np.full((2, 6), 7, dtype=np.int32), np.full(6, 7, dtype=np.int32)]
        out += [np.full((2, 2), 7, dtype=np.int64) for _ in range(2)]
        rc = L.sgdml_b200_remd_run(handle, n_temps, kT.ctypes.data, n_steps, dt, gamma, 0, every, stride,
                                   *(x.ctypes.data for x in out), _lib.current_stream())
        return rc, out

    rc, out = call(rex._handle)
    assert rc <= -1000  # no state yet
    rex._set_state_raw(R0, V0, step=7)
    rex._run_raw(4, dt, 1.0, kT, 1)
    before = rex._get_state_raw()
    bad = [dict(n_temps=1), dict(n_temps=4), dict(n_temps=0), dict(n_temps=-3), dict(kT=[kT[0], 0.0, kT[2]]),
           dict(kT=[kT[0], -1.0, kT[2]]), dict(kT=[kT[0], np.nan, kT[2]]), dict(kT=[np.inf, kT[1], kT[2]]),
           dict(gamma=0.0), dict(gamma=-1.0), dict(gamma=np.nan), dict(every=-1), dict(stride=3), dict(stride=-1),
           dict(dt=0.0), dict(dt=np.nan), dict(n_steps=-1)]
    for kw in bad:
        rc, out = call(h, **kw)
        assert rc <= -1000, kw
        assert all(np.all(x == (1.5 if x.dtype == np.float64 else 7)) for x in out), kw
    assert L.sgdml_b200_remd_run(None, 3, np.asarray(kT).ctypes.data, 10, dt, 1.0, 0, 1, 0, *([None] * 8),
                                 None) <= -1000
    assert L.sgdml_b200_remd_run(h, 3, None, 10, dt, 1.0, 0, 1, 0, *([None] * 8), None) <= -1000
    # a ring-polymer handle holds no ladders
    pimd = sgdml_b200.GDMLPathIntegralDynamics(gp, md_fs_masses(np.ones(gp.n_atoms)), 3, n_polymers=2, E_to_eV=1.0,
                                               F_to_eV_Ang=1.0)
    pimd._set_state_raw(R0)
    assert call(pimd._handle)[0] <= -1000
    assert _same(before, rex._get_state_raw())
    with pytest.raises(ValueError):
        rex._run_raw(4, dt, 1.0, kT[:2], 1)


@pytest.mark.gpu
def test_canonical_ensemble_at_every_slot(spring_task):  # noqa: F811
    """256 ladders of 4 temperatures on a trained harmonic spring model, exchanging every 5 steps: at every slot
    <E_kin> is (3N/2) kT_k and <E_pot> agrees with plain Langevin at kT_k, each within 5 block standard errors (fixed
    seeds)."""
    import sgdml_b200

    model = sgdml_b200.GDMLTrain().train(spring_task)
    gp = sgdml_b200.GDMLPredict(model)
    s = np.full(15, 0.1)
    masses = md_fs_masses(1.0 / s[::3])
    kT = np.geomspace(0.01, 0.03375, 4)  # neighbours 1.5 apart
    n_lad, dt, gamma = 256, 0.05, 1.0
    R0 = np.tile(synth_base(), (n_lad * 4, 1))
    rex = sgdml_b200.GDMLReplicaExchange(gp, masses, np.ones(4), n_ladders=n_lad, E_to_eV=1.0, F_to_eV_Ang=1.0)
    rex._set_state_raw(R0)
    rex._run_raw(1000, dt, gamma, kT, 5, seed=31)
    fr = rex._run_raw(2000, dt, gamma, kT, 5, seed=31, stride=10, frames=('E_pot', 'E_kin'))
    acc = fr['n_accepted'].sum(0) / fr['n_attempted'].sum(0)
    print('acceptance per pair: %s' % acc)
    assert np.all(acc > 0.1)

    def mean_se(series):  # (n_frames,) -> mean and standard error of 10 block means
        blocks = series.reshape(10, -1).mean(1)
        return series.mean(), blocks.std(ddof=1) / np.sqrt(len(blocks))

    Ek = fr['E_kin'].reshape(-1, n_lad, 4).mean(1)
    Ep = fr['E_pot'].reshape(-1, n_lad, 4).mean(1)
    for k in range(4):
        m, se = mean_se(Ek[:, k])
        want = 1.5 * 5 * kT[k]
        print('slot %d: <E_kin> %.6g, (3N/2) kT %.6g, se %.3g' % (k, m, want, se))
        assert abs(m - want) < 5.0 * se
        md = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=n_lad, E_to_eV=1.0, F_to_eV_Ang=1.0)
        md._set_state_raw(R0[:n_lad])
        md._run_raw(1000, dt, gamma, kT[k], seed=40 + k)
        plain = md._run_raw(2000, dt, gamma, kT[k], seed=40 + k, stride=10, frames=('E_pot',))['E_pot'].mean(1)
        m1, se1 = mean_se(Ep[:, k])
        m2, se2 = mean_se(plain)
        print('slot %d: <E_pot> %.6g (se %.3g), plain Langevin %.6g (se %.3g)' % (k, m1, se1, m2, se2))
        assert abs(m1 - m2) < 5.0 * np.hypot(se1, se2)


def synth_base():
    from sgdml_b200 import synth

    return synth.base_geometry(5).reshape(1, -1)


@pytest.mark.gpu
def test_crosses_a_barrier_that_plain_langevin_does_not():
    """A model trained on the double-well hinge of test_neb.py (barrier 0.1): the lowest slot of a ladder from kT 0.006
    up to the barrier height visits both wells; plain Langevin at kT 0.006 from the same well, 8 replicas for the same
    steps, stays in it."""
    import sgdml_b200
    from test_neb import _DW_DC, _DW_PHI, _dw_hinge, _dw_task

    model = sgdml_b200.GDMLTrain().train(_dw_task())
    gp = sgdml_b200.GDMLPredict(model)
    masses = md_fs_masses(np.ones(4))
    kT = np.geomspace(0.006, 0.1, 8)
    A = _dw_hinge(_DW_PHI[0]).reshape(1, 12)
    dt, gamma, n = 0.02, 1.0, 10000

    def d01(R):
        X = R.reshape(R.shape[0], -1, 4, 3)
        return np.linalg.norm(X[..., 0, :] - X[..., 1, :], axis=-1)

    rex = sgdml_b200.GDMLReplicaExchange(gp, masses, np.ones(8), E_to_eV=1.0, F_to_eV_Ang=1.0)
    rex._set_state_raw(np.repeat(A, 8, 0))
    fr = rex._run_raw(n, dt, gamma, kT, 2, seed=5, stride=10, frames=('R', 'walker'))
    low = d01(fr['R'])[:, 0]
    print('REMD: acceptance %s, lowest slot in the far well %.3f of the time, walkers there %s' % (
        fr['n_accepted'][0] / fr['n_attempted'][0], (low > _DW_DC).mean(), np.unique(fr['walker'][:, 0])))
    assert (low < _DW_DC).any() and (low > _DW_DC).any()

    md = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=8, E_to_eV=1.0, F_to_eV_Ang=1.0)
    md._set_state_raw(np.repeat(A, 8, 0))
    plain = d01(md._run_raw(n, dt, gamma, kT[0], seed=6, stride=10, frames=('R',))['R'])
    print('plain Langevin: d01 in [%.3f, %.3f], barrier at %.3f' % (plain.min(), plain.max(), _DW_DC))
    assert np.all(plain < _DW_DC)
