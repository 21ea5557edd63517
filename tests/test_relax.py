"""Geometry optimisation on the device (sgdml_b200_relax_*, sgdml_b200.GDMLRelaxation) against the NumPy restatement
of tests/relax_oracle.py driven by GDMLPredict.predict: every predictor form, convergence counts, freezing, graph
against plain launches, block lengths, chunking, batch independence, int8 slices, isolation from the predictor's own
calls and from MD, quenching Langevin frames of a trained spring model, public units and argument errors.
"""

import numpy as np
import pytest

import relax_oracle
from conftest import rel_err
from md_common import FIXTURES_MD, _N_SPRING, _cuda_forces, _spring_pes, md_fs_masses, spring_task  # noqa: F401

pytestmark = pytest.mark.gpu


def _setup(name, n_rep=3, chunk=0, slices=0):
    """(GDMLPredict, GDMLRelaxation in model units, R0 (n_rep, 3N), optimiser scales (fire dt, lbfgs h0, maxstep))."""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    gp = sgdml_b200.GDMLPredict(model)
    if slices:
        gp.set_contraction_slices(slices)
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=n_rep, E_to_eV=1.0, F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    R0 = np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)
    R0 = R0[np.arange(n_rep) % R0.shape[0]].copy()
    if n_rep > Rq.shape[0]:
        R0 += 1e-2 * np.random.default_rng(1).standard_normal(R0.shape)
    _, F0 = gp.predict(R0)
    f = float(np.max(np.abs(F0)))
    return gp, rel, R0, {'dt': float(np.sqrt(0.01 / f)), 'h0': 0.01 / f, 'maxstep': 0.05}


def _device(rel, R0, opt, steps, fmax, sc, memory=8):
    rel._set_state_raw(R0)
    if opt == 'fire':
        n, c, fm = rel._relax_raw('fire', steps, fmax, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    else:
        n, c, fm = rel._relax_raw('lbfgs', steps, fmax, sc['maxstep'], memory, sc['h0'])
    st = rel._get_state_raw()
    return {'R': st['R'], 'F': st['F'], 'E': st['E_pot'], 'V': st['V'], 'step': st['step'], 'n_steps': n,
            'converged': c.astype(bool), 'fmax': fm}


def _oracle(gp, R0, opt, steps, fmax, sc, memory=8):
    forces = _cuda_forces(gp)
    if opt == 'fire':
        return relax_oracle.fire(forces, R0, steps, fmax, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    return relax_oracle.lbfgs(forces, R0, steps, fmax, sc['maxstep'], memory, sc['h0'])


def _same(a, b, keys=('R', 'F', 'E', 'n_steps', 'converged', 'fmax')):
    return all(np.array_equal(a[k], b[k]) for k in keys)


def _tie_free_fmax(gp, R0, opt, steps, sc):
    """A threshold between the replicas' max |F| after 2/3 of `steps` (so that some converge well before the end), at
    least 1e-6 (relative) from every value the convergence test compares with it; and the oracle's run at that
    threshold."""
    ref = _oracle(gp, R0, opt, 2 * steps // 3, 0.0, sc)
    f = np.sort(ref['fmax'])
    fmax = float(np.sqrt(f[len(f) // 2 - 1] * f[len(f) // 2]))
    for _ in range(50):
        out = _oracle(gp, R0, opt, steps, fmax, sc)
        if np.min(np.abs(out['tested'] / fmax - 1.0)) > 1e-6:
            return fmax, out
        fmax *= 1.0 + 1e-4
    raise AssertionError('no tie-free threshold')


# ---------------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_matches_restatement(name, opt):
    gp, rel, R0, sc = _setup(name)
    dev = _device(rel, R0, opt, 12, 0.0, sc)
    ref = _oracle(gp, R0, opt, 12, 0.0, sc)
    print('%s %s: R bit-identical to the restatement: %s' % (name, opt, np.array_equal(dev['R'], ref['R'])))
    assert rel_err(dev['R'], ref['R']) < 1e-12
    assert rel_err(dev['E'], ref['E']) < 1e-12
    assert np.all(dev['n_steps'] == 12) and not dev['converged'].any()
    assert rel_err(dev['fmax'], ref['fmax']) < 1e-12
    assert np.all(dev['V'] == 0.0) and dev['step'] == 0
    assert rel_err(dev['R'], R0) > 1e-6  # it moved


@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
def test_convergence_matches_restatement(opt):
    gp, rel, R0, sc = _setup('n9_m16_s6', n_rep=6)
    fmax, ref = _tie_free_fmax(gp, R0, opt, 40, sc)
    dev = _device(rel, R0, opt, 40, fmax, sc)
    print('%s: fmax %.6g, steps %s, converged %s' % (opt, fmax, dev['n_steps'].tolist(), dev['converged'].tolist()))
    assert np.array_equal(dev['n_steps'], ref['n_steps'])
    assert np.array_equal(dev['converged'], ref['converged'])
    assert dev['converged'].any() and dev['n_steps'].min() < dev['n_steps'].max()
    assert rel_err(dev['R'], ref['R']) < 1e-12
    # a fresh prediction at every converged replica's positions
    _, F = gp.predict(dev['R'])
    f = np.sqrt((F.reshape(len(F), -1, 3) ** 2).sum(-1)).max(1)
    assert np.all(f[dev['converged']] < fmax)
    assert np.all(f[~dev['converged']] >= fmax)


@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
def test_second_call_on_converged_replicas(opt):
    gp, rel, R0, sc = _setup('n12_m8_s12', n_rep=4)
    fmax = 0.05 * float(np.max(np.abs(gp.predict(R0)[1])))
    first = _device(rel, R0, opt, 2000, fmax, sc)
    assert first['converged'].all(), first['fmax']
    before = rel._get_state_raw()
    n, c, fm = (rel._relax_raw('fire', 100, fmax, sc['maxstep'], sc['dt'], 10.0 * sc['dt']) if opt == 'fire' else
                rel._relax_raw('lbfgs', 100, fmax, sc['maxstep'], 8, sc['h0']))
    assert np.all(n == 0) and np.all(c == 1) and np.array_equal(fm, first['fmax'])
    after = rel._get_state_raw()
    assert all(np.array_equal(before[k], after[k]) for k in before)


@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12', 'pbc_n6_m8'])
def test_graph_blocks_and_chunks(name, opt, monkeypatch):
    from sgdml_b200 import _lib

    gp, rel, R0, sc = _setup(name, n_rep=5)
    fmax, _ = _tie_free_fmax(gp, R0, opt, 30, sc)
    a = _device(rel, R0, opt, 30, fmax, sc)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _device(rel, R0, opt, 30, fmax, sc)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    for block in (1, 7, 1000):
        _lib.check(_lib.lib().sgdml_b200_set_relax_block(block), 'set_relax_block')
        try:
            c = _device(rel, R0, opt, 30, fmax, sc)
        finally:
            _lib.lib().sgdml_b200_set_relax_block(0)
        assert _same(a, c), block
    _, rc, _, _ = _setup(name, n_rep=5, chunk=2)
    d = _device(rc, R0, opt, 30, fmax, sc)
    assert np.array_equal(d['n_steps'], a['n_steps']) and np.array_equal(d['converged'], a['converged'])
    for k in ('R', 'E', 'fmax'):
        assert rel_err(d[k], a[k]) < 1e-12, k


@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
def test_replica_alone_and_in_batch(opt):
    import sgdml_b200

    gp, rel, R0, sc = _setup('n21_m6_s6', n_rep=4)
    batch = _device(rel, R0, opt, 15, 0.0, sc)
    one = sgdml_b200.GDMLRelaxation(gp, n_replicas=1, E_to_eV=1.0, F_to_eV_Ang=1.0)
    alone = _device(one, R0[2:3], opt, 15, 0.0, sc)
    assert rel_err(alone['R'][0], batch['R'][2]) < 1e-12
    assert rel_err(alone['E'][0], batch['E'][2]) < 1e-12


@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
def test_int8_slices(opt):
    gp, rel, R0, sc = _setup('big_n100_m2_s12', slices=6)
    dev = _device(rel, R0, opt, 12, 0.0, sc)
    ref = _oracle(gp, R0, opt, 12, 0.0, sc)
    assert rel_err(dev['R'], ref['R']) < 1e-12
    assert rel_err(dev['E'], ref['E']) < 1e-12


def test_isolated_from_predict_calls_and_md():
    import torch

    import md_oracle
    import sgdml_b200

    gp, rel, R0, sc = _setup('n12_m8_s12')
    ref = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    a = _device(ref, R0, 'lbfgs', 10, 0.0, sc)
    a2 = _device(ref, R0, 'fire', 10, 0.0, sc)

    Rbig = np.tile(R0, (30, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((90, R0.shape[1]))
    E_before, F_before = gp.predict(Rbig)
    rel._set_state_raw(R0, step=7)
    gp.predict(Rbig)
    gp.predict_hvp(Rbig, np.ones_like(Rbig))
    gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (90, 1, 1)))
    n, c, fm = rel._relax_raw('lbfgs', 10, 0.0, sc['maxstep'], 8, sc['h0'])
    st = rel._get_state_raw()
    assert np.array_equal(st['R'], a['R']) and np.array_equal(st['E_pot'], a['E']) and np.array_equal(fm, a['fmax'])
    assert st['step'] == 7 and np.all(st['V'] == 0.0)
    gp.predict(Rbig)
    b2 = _device(rel, R0, 'fire', 10, 0.0, sc)
    assert _same(a2, b2)
    E_after, F_after = gp.predict(Rbig)
    assert np.array_equal(E_before, E_after) and np.array_equal(F_before, F_after)

    # MD continues from the relaxed positions, at rest, with the step counter where it was
    rel._set_state_raw(R0, step=7)
    rel._relax_raw('lbfgs', 10, 0.0, sc['maxstep'], 8, sc['h0'])
    dt = 0.5 * sc['dt']
    fr = rel._run_raw(5, dt, stride=5)
    s = np.ones(R0.shape[1])
    _, want = md_oracle.run(_cuda_forces(gp), a['R'], np.zeros_like(R0), s, 5, dt, stride=5)
    assert rel_err(fr['R'], want['R']) < 1e-12
    assert rel._get_state_raw()['step'] == 12


def _pair_distances(R):
    X = np.asarray(R).reshape(-1, _N_SPRING, 3)
    return np.sqrt(((X[:, :, None] - X[:, None]) ** 2).sum(-1))


@pytest.mark.parametrize('opt', ['lbfgs', 'fire'])
def test_quench_langevin_frames(spring_task, opt):  # noqa: F811
    """Quench Langevin frames of the spring model trained in the test: every frame converges, its energy falls, and it
    ends at the spring minimum (the pair distances d0) within the model's accuracy."""
    import sgdml_b200
    from sgdml_b200 import synth

    model = sgdml_b200.GDMLTrain().train(spring_task)
    gp = sgdml_b200.GDMLPredict(model)
    dyn = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.full(_N_SPRING, 10.0)), n_replicas=8, E_to_eV=1.0,
                                  F_to_eV_Ang=1.0)
    r0 = synth.base_geometry(_N_SPRING).reshape(1, -1)
    dt = 0.02 / np.sqrt(4.0 * 2.0 * 0.1)
    dyn._set_state_raw(np.tile(r0, (8, 1)))
    fr = dyn._run_raw(400, dt, 0.05 / dt, 0.02, seed=3, stride=100, frames=('R', 'E_pot'))
    frames = fr['R'].reshape(-1, 3 * _N_SPRING)
    E_frames = fr['E_pot'].ravel()
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=len(frames), E_to_eV=1.0, F_to_eV_Ang=1.0)
    out = rel.relax(frames.reshape(-1, _N_SPRING, 3), fmax=1e-4, max_steps=3000, optimizer=opt, maxstep=0.1,
                    alpha=10.0, dt=0.1, dtmax=0.5)
    d0 = _pair_distances(r0)[0]
    dev = np.abs(_pair_distances(out['positions']) - d0).max((1, 2))
    E_true_frames = _spring_pes(frames)[0]
    E_true = _spring_pes(out['positions'])[0]
    print('%s: steps %d..%d, max |d - d0| %.2e, true E %.2e of the frames\' %.2e' % (
        opt, out['n_steps'].min(), out['n_steps'].max(), dev.max(), E_true.max(), E_true_frames.mean()))
    assert out['converged'].all() and np.all(out['fmax'] < 1e-4)
    assert np.all(out['potential_energy'] < E_frames)
    assert dev.max() < 0.05
    assert np.all(E_true < 0.05 * E_true_frames.mean())


def test_public_units():
    """GDMLRelaxation in eV / Angstrom (a kcal/mol model, the default units) against its model-unit form, and CUDA
    tensors in and out."""
    import torch

    import hvp_oracle
    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc

    model, Rq, _ = hvp_oracle.fixture_model('n9_m16_s6')
    rel = sgdml_b200.GDMLRelaxation(model, n_replicas=2)
    R0 = np.asarray(Rq[:2], dtype=np.float64).reshape(2, 9, 3)
    out = rel.relax(R0, fmax=0.0, max_steps=10, optimizer='lbfgs', memory=5, alpha=35.0, maxstep=0.1)
    raw = sgdml_b200.GDMLRelaxation(rel.gdml_predict, n_replicas=2)
    raw._set_state_raw(R0.reshape(2, -1))
    n, c, fm = raw._relax_raw('lbfgs', 10, 0.0, 0.1, 5, kc / 35.0)
    st = raw._get_state_raw()
    assert np.array_equal(out['positions'], st['R'].reshape(2, 9, 3))
    assert np.allclose(out['potential_energy'], st['E_pot'] * kc, rtol=1e-15)
    assert np.allclose(out['fmax'], fm * kc, rtol=1e-15) and np.array_equal(out['n_steps'], n)
    assert out['forces'].shape == (2, 9, 3) and out['converged'].dtype == bool
    fire = rel.relax(R0, fmax=0.0, max_steps=10, optimizer='fire', dt=0.2, dtmax=0.8)
    raw._set_state_raw(R0.reshape(2, -1))
    raw._relax_raw('fire', 10, 0.0, 0.2, 0.2 * np.sqrt(kc), 0.8 * np.sqrt(kc))
    assert np.array_equal(fire['positions'], raw._get_state_raw()['R'].reshape(2, 9, 3))
    t = rel.relax(torch.from_numpy(R0).cuda(), fmax=0.0, max_steps=10, optimizer='lbfgs', memory=5, alpha=35.0,
                  maxstep=0.1)
    assert t['positions'].is_cuda and t['n_steps'].is_cuda
    assert np.array_equal(t['positions'].cpu().numpy(), out['positions'])
    # positions=None re-relaxes the current state
    again = rel.relax(fmax=0.0, max_steps=3)
    assert not np.array_equal(again['positions'].cpu().numpy(), out['positions'])


def test_bad_input_is_rejected():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, rel, R0, sc = _setup('n9_m16_s6')
    L = _lib.lib()
    h = rel._handle
    fresh = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    assert L.sgdml_b200_relax_fire(fresh._handle, 10, 0.0, 0.1, 0.1, 1.0, None, None, None, None) <= -1000  # no state
    assert L.sgdml_b200_relax_lbfgs(fresh._handle, 10, 0.0, 0.1, 5, 0.1, None, None, None, None) <= -1000
    rel._set_state_raw(R0, step=3)
    rel._relax_raw('lbfgs', 4, 0.0, 0.05, 4, sc['h0'])
    before = rel._get_state_raw()
    fire_bad = [dict(max_steps=-1), dict(fmax=-1.0), dict(fmax=np.nan), dict(fmax=np.inf), dict(maxstep=0.0),
                dict(maxstep=np.nan), dict(dt=0.0), dict(dt=-1.0), dict(dt=np.inf), dict(dtmax=0.0),
                dict(dtmax=np.nan)]
    lbfgs_bad = [dict(max_steps=-1), dict(fmax=-1.0), dict(fmax=np.nan), dict(maxstep=-0.1), dict(maxstep=np.inf),
                 dict(memory=0), dict(memory=33), dict(h0=0.0), dict(h0=-1.0), dict(h0=np.nan)]
    for kw in fire_bad:
        a = dict(max_steps=10, fmax=0.0, maxstep=0.1, dt=0.1, dtmax=1.0)
        a.update(kw)
        out = (np.full(3, 7, dtype=np.int64), np.full(3, 7, dtype=np.int32), np.full(3, 7.0))
        rc = L.sgdml_b200_relax_fire(h, a['max_steps'], a['fmax'], a['maxstep'], a['dt'], a['dtmax'],
                                     *(x.ctypes.data for x in out), _lib.current_stream())
        assert rc <= -1000, kw
        assert all(np.all(x == 7) for x in out)
    for kw in lbfgs_bad:
        a = dict(max_steps=10, fmax=0.0, maxstep=0.1, memory=5, h0=0.1)
        a.update(kw)
        out = (np.full(3, 7, dtype=np.int64), np.full(3, 7, dtype=np.int32), np.full(3, 7.0))
        rc = L.sgdml_b200_relax_lbfgs(h, a['max_steps'], a['fmax'], a['maxstep'], a['memory'], a['h0'],
                                      *(x.ctypes.data for x in out), _lib.current_stream())
        assert rc <= -1000, kw
        assert all(np.all(x == 7) for x in out)
    assert L.sgdml_b200_relax_fire(None, 10, 0.0, 0.1, 0.1, 1.0, None, None, None, None) <= -1000
    assert L.sgdml_b200_set_relax_block(-1) <= -1000
    after = rel._get_state_raw()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    with pytest.raises(ValueError):
        rel.relax(optimizer='newton')
    # memory grows on a later call and the results follow the restatement
    dev = _device(rel, R0, 'lbfgs', 12, 0.0, sc, memory=32)
    ref = _oracle(gp, R0, 'lbfgs', 12, 0.0, sc, memory=32)
    assert rel_err(dev['R'], ref['R']) < 1e-12
