"""The NumPy restatement of the device optimisers (tests/relax_oracle.py) on analytic surfaces, and the CPU side of
sgdml_b200_relax_* / sgdml_b200.GDMLRelaxation: the restated FIRE and L-BFGS relax the harmonic-spring surface of
test_md.py to its pair distances, FIRE's first step, the step caps, the L-BFGS history resets, the loud failure without
a device and the bound entry points.
"""

import os

import numpy as np
import pytest

import relax_oracle
from md_common import _N_SPRING, _spring_pes

_EPS = np.finfo(np.float64).eps


def _pair_distances(R):
    X = np.asarray(R).reshape(-1, _N_SPRING, 3)
    return np.sqrt(((X[:, :, None] - X[:, None]) ** 2).sum(-1))


def _spring_start(n_rep=4, scale=0.15, seed=0):
    from sgdml_b200 import synth

    r0 = synth.base_geometry(_N_SPRING).reshape(1, -1)
    return r0 + scale * np.random.default_rng(seed).standard_normal((n_rep, r0.shape[1])), r0


def test_block_sum_order():
    """128 strided partials, then the tree: exact on integers, and not NumPy's pairwise sum on a cancelling vector."""
    x = np.arange(1.0, 301.0)
    assert relax_oracle.block_sum(x) == x.sum()
    y = np.zeros(256)
    y[0], y[128], y[1] = 1.0, 1e16, -1e16
    # thread 0 adds 1 + 1e16 (rounds to 1e16), thread 1 holds -1e16: the tree gives 0
    assert relax_oracle.block_sum(y) == 0.0
    assert relax_oracle.block_sum(np.stack([y, x[:256]])).tolist() == [0.0, x[:256].sum()]


@pytest.mark.parametrize('opt', ['fire', 'lbfgs'])
def test_restatement_relaxes_springs(opt):
    R0, r0 = _spring_start()
    d0 = _pair_distances(r0)[0]
    if opt == 'fire':
        out = relax_oracle.fire(_spring_pes, R0, 5000, 1e-8, 0.2, 0.1, 1.0)
    else:
        out = relax_oracle.lbfgs(_spring_pes, R0, 5000, 1e-8, 0.2, 20, 0.1)
    assert out['converged'].all(), out['fmax']
    assert np.all(out['fmax'] < 1e-8)
    E, F = _spring_pes(out['R'])
    assert np.array_equal(E, out['E']) and np.array_equal(F.reshape(out['F'].shape), out['F'])
    err = np.max(np.abs(_pair_distances(out['R']) - d0))
    print('%s: steps %s, max |d - d0| %.2e' % (opt, out['n_steps'].tolist(), err))
    assert err < 1e-7
    assert np.all(E < 1e-14)


def test_fire_first_step_skips_mixing_and_keeps_dt():
    R0, _ = _spring_start(n_rep=1, scale=0.01)
    F0 = _spring_pes(R0)[1].reshape(R0.shape)
    dt = 0.1
    out = relax_oracle.fire(_spring_pes, R0, 1, 0.0, 10.0, dt, 1.0)
    assert np.array_equal(out['R'], R0 + dt * (dt * F0))  # v = 0 + dt F, dr = dt v, no cap
    assert out['dt'][0] == dt and out['alpha'][0] == 0.1 and out['n_pos'][0] == 0
    assert out['n_steps'][0] == 1
    # the second step mixes (F.v > 0 from rest) and counts a positive step
    two = relax_oracle.fire(_spring_pes, R0, 2, 0.0, 10.0, dt, 1.0)
    assert two['n_pos'][0] == 1 and two['dt'][0] == dt


def test_fire_cap_is_hit_exactly():
    R0, _ = _spring_start(n_rep=3, scale=0.4, seed=4)
    maxstep = 1e-3
    out = relax_oracle.fire(_spring_pes, R0, 1, 0.0, maxstep, 0.5, 1.0)
    step = np.sqrt(((out['R'] - R0) ** 2).sum(1))
    # |dr| = maxstep up to the rounding of r + dr
    assert np.all(np.abs(step - maxstep) <= 4 * _EPS * np.abs(R0).max()), step - maxstep


def test_lbfgs_cap_is_hit_exactly():
    R0, _ = _spring_start(n_rep=3, scale=0.4, seed=5)
    maxstep = 1e-3
    out = relax_oracle.lbfgs(_spring_pes, R0, 1, 0.0, maxstep, 5, 1.0)
    per_atom = np.sqrt(((out['R'] - R0).reshape(3, -1, 3) ** 2).sum(-1)).max(1)
    assert np.all(np.abs(per_atom - maxstep) <= 4 * _EPS * np.abs(R0).max()), per_atom - maxstep


def _double_well(R):
    """Sum over coordinates of (x^2 - 1)^2: concave for |x| < 1/sqrt(3)."""
    R = np.asarray(R)
    x2 = R * R
    return ((x2 - 1.0) ** 2).sum(1), -4.0 * R * (x2 - 1.0)


def test_lbfgs_clears_history_on_negative_curvature():
    R0 = np.full((1, 3), 0.1)  # near the barrier top: every step downhill, s.y < 0 while in the concave region
    out = relax_oracle.lbfgs(_double_well, R0, 200, 1e-8, 0.2, 10, 0.05)
    used = out['n_hist'][:, 0]
    print('pairs per step:', used[:20].tolist())
    assert used[0] == 0 and used[1] == 0  # first step, then the rejected pair (s.y < 0)
    E = [_double_well(R0)[0][0]]
    assert np.all(out['E'] < E[0])
    assert used.max() >= 2  # the history builds again in the convex well
    assert out['converged'][0] and np.allclose(np.abs(out['R']), 1.0, atol=1e-8)
    # the same walk in the convex region keeps its first pair
    conv = relax_oracle.lbfgs(_double_well, np.full((1, 3), 0.8), 3, 0.0, 0.2, 10, 0.05)
    assert conv['n_hist'][1, 0] == 1


def _bowl(R):
    R = np.asarray(R)
    return 0.5 * (R * R).sum(1), -R


def test_lbfgs_clears_history_on_energy_rise():
    R0 = np.ones((1, 3))
    # h0 = 3 overshoots to -2 R0: s.y > 0, but E rises, so the pair is dropped
    rise = relax_oracle.lbfgs(_bowl, R0, 2, 0.0, 100.0, 5, 3.0)
    assert rise['n_hist'][1, 0] == 0
    # h0 = 1.5 lands at -R0 / 2: E falls and the pair is kept
    fall = relax_oracle.lbfgs(_bowl, R0, 2, 0.0, 100.0, 5, 1.5)
    assert fall['n_hist'][1, 0] == 1


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_relaxation_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLRelaxation({'type': 'm'})
    L = _lib.lib()
    assert L.sgdml_b200_relax_fire(None, 10, 0.05, 0.2, 0.1, 1.0, None, None, None, None) == -1002
    assert L.sgdml_b200_relax_lbfgs(None, 10, 0.05, 0.2, 20, 0.01, None, None, None, None) == -1002


def test_relax_entry_points_are_bound():
    import sgdml_b200
    from sgdml_b200 import _lib

    for name in ('sgdml_b200_relax_fire', 'sgdml_b200_relax_lbfgs', 'sgdml_b200_set_relax_block'):
        assert name in _lib.SIGNATURES
        getattr(_lib.lib(), name)
    assert sgdml_b200.GDMLRelaxation.relax


def test_unknown_optimizer_is_rejected():
    from sgdml_b200.md import GDMLRelaxation

    r = GDMLRelaxation.__new__(GDMLRelaxation)
    with pytest.raises(ValueError, match='optimizer'):
        r.relax(optimizer='bfgs')


def test_relaxation_has_no_md_run():
    """The relaxation handle's unit inverse masses are no masses: MD goes through GDMLDynamics."""
    from sgdml_b200.md import GDMLRelaxation

    r = GDMLRelaxation.__new__(GDMLRelaxation)
    with pytest.raises(TypeError, match='GDMLDynamics'):
        r.run(10, 0.5)
