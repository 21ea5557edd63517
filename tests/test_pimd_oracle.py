"""The NumPy restatement of the ring-polymer integrator (tests/pimd_oracle.py) on the CPU: the normal-mode matrix, the
free ring-polymer rotation, the one-bead limit against tests/md_oracle.py, and the quantum statistics of a harmonic
oscillator, which the restatement must reproduce before the device is compared against it.  Also the loud failure of
GDMLPathIntegralDynamics without a device."""

import ctypes
import os

import numpy as np
import pytest

import md_oracle
import pimd_oracle


@pytest.mark.parametrize('P', [1, 2, 3, 4, 7, 8, 32, 64])
def test_normal_modes_are_orthonormal(P):
    C = pimd_oracle.normal_modes(P)
    tol = 4 * P * np.finfo(float).eps  # P-term dot products
    assert np.max(np.abs(C.T @ C - np.eye(P))) < tol
    assert np.max(np.abs(C @ C.T - np.eye(P))) < tol
    if P == 1:
        assert np.array_equal(C, np.ones((1, 1)))


def test_free_ring_rotation_is_exact_and_reversible():
    """With zero force the A steps rotate every normal mode exactly: after n steps of dt, mode k has turned by
    omega_k n dt (the centroid drifts freely), and reversing the velocities brings the polymer back."""
    P, n_poly, dimi, n, dt = 8, 2, 6, 40, 0.3
    kT, hbar = 0.7, 0.9
    s = np.linspace(0.5, 2.0, dimi)
    rng = np.random.default_rng(0)
    R0 = rng.standard_normal((n_poly, P, dimi))
    V0 = rng.standard_normal((n_poly, P, dimi))

    def zero(R):
        return np.zeros(R.shape[0]), np.zeros_like(R)

    (R1, V1, _, _), _ = pimd_oracle.run(zero, R0, V0, s, n, dt, kT, hbar)
    t = pimd_oracle.constants(P, dt, kT, hbar, 0.0, 0.0, s)
    C = t['C']
    q0, u0 = pimd_oracle.to_modes(C, R0), pimd_oracle.to_modes(C, V0)
    w = t['w'][:, None]
    tt = n * dt
    ws = np.where(w > 0, w, 1.0)
    q = np.where(w > 0, q0 * np.cos(w * tt) + u0 * np.sin(w * tt) / ws, q0 + u0 * tt)
    u = np.where(w > 0, -q0 * ws * np.sin(w * tt) + u0 * np.cos(w * tt), u0)
    assert np.max(np.abs(R1 - pimd_oracle.from_modes(C, q))) < 1e-12
    assert np.max(np.abs(V1 - pimd_oracle.from_modes(C, u))) < 1e-12
    # the tables are the closed form
    assert np.allclose(t['cos'], np.cos(t['w'] * 0.5 * dt), rtol=0, atol=1e-16)
    assert np.allclose(t['msin'], -t['w'] * np.sin(t['w'] * 0.5 * dt), rtol=1e-15, atol=0)
    (R2, V2, _, _), _ = pimd_oracle.run(zero, R1, -V1, s, n, dt, kT, hbar)
    assert np.max(np.abs(R2 - R0)) < 1e-12
    assert np.max(np.abs(-V2 - V0)) < 1e-12


def _anharmonic(R):
    E = (0.5 * R * R + 0.1 * R**4).sum(-1)
    return E, -(R + 0.4 * R**3)


@pytest.mark.parametrize('gamma', [0.0, 0.3])
def test_one_bead_is_the_classical_integrator(gamma):
    """P = 1 is md_oracle.run bit for bit, noise included, with any hbar and lambda."""
    n_poly, dimi, n, dt = 3, 7, 25, 0.05
    s = np.linspace(0.5, 2.0, dimi)
    rng = np.random.default_rng(1)
    R0, V0 = rng.standard_normal((n_poly, dimi)), rng.standard_normal((n_poly, dimi))
    kT = 0.8 if gamma > 0 else 0.0
    seed, step0 = (5 << 32) + 9, (1 << 32) - 7
    (R, V, F, E), fr = md_oracle.run(_anharmonic, R0, V0, s, n, dt, gamma, kT, seed, step0, stride=5)
    (Rp, Vp, Fp, Ep), fp = pimd_oracle.run(_anharmonic, R0[:, None], V0[:, None], s, n, dt, kT, 1.3, gamma, 0.7,
                                           seed, step0, stride=5)
    assert np.array_equal(Rp[:, 0], R) and np.array_equal(Vp[:, 0], V)
    assert np.array_equal(fp['R'][:, :, 0], fr['R']) and np.array_equal(fp['V'][:, :, 0], fr['V'])
    assert np.allclose(fp['E_kin'][:, :, 0], fr['E_kin'], rtol=1e-14, atol=0)
    # one bead: K_prim = K_cv = 3N kT / 2 exactly
    assert np.all(fp['K_prim'] == 0.5 * dimi * kT) and np.all(fp['K_cv'] == 0.5 * dimi * kT)


# A 3-D isotropic harmonic oscillator (m = 1, omega = 1, hbar = 1) at beta hbar omega = 4 with P = 8 beads: the exact
# finite-P <V>, <K_prim> and <K_cv> are 3 x pimd_oracle.harmonic_value = 0.7559 (classical: 3 kT / 2 = 0.375; the
# P -> infinity limit 3 hbar omega coth(2) / 4 = 0.7780).  PILE-L at lambda = 1 with centroid friction omega, dt = 0.05
# (omega dt = 0.05; the free ring-polymer part, omega_k up to 4, is integrated exactly).  _HARMONIC_BIAS_BOUND bounds
# the integrator's bias: the exact stationary covariance of the step as a linear map, below.
_HO = dict(P=8, kT=0.25, hbar=1.0, omega=1.0, dt=0.05, gamma=1.0, lam=1.0)


def _harmonic(R):
    return 0.5 * (R * R).sum(-1), -R


def _step_map(P, dimi):
    """The step of one polymer with a harmonic force as z' = A z + B xi, z = (x, v full-step) of every bead (one
    coordinate: the oscillator is isotropic), from the restatement's own pieces."""
    c = _HO
    t = pimd_oracle.constants(P, c['dt'], c['kT'], c['hbar'], c['gamma'], c['lam'], np.ones(1))
    h = t['h']

    def step(x, v, xi):
        v = v + h * (-x)
        q, u = pimd_oracle.to_modes(t['C'], x[None, :, None]), pimd_oracle.to_modes(t['C'], v[None, :, None])
        q, u = pimd_oracle.free_ring(t, q, u)
        u = t['c1'][:, None] * u + t['sigma'] * xi[None, :, None]
        q, u = pimd_oracle.free_ring(t, q, u)
        x, v = pimd_oracle.from_modes(t['C'], q)[0, :, 0], pimd_oracle.from_modes(t['C'], u)[0, :, 0]
        return x, v + h * (-x)

    A = np.zeros((2 * P, 2 * P))
    B = np.zeros((2 * P, P))
    for i in range(2 * P):
        z = np.eye(2 * P)[i]
        x, v = step(z[:P], z[P:], np.zeros(P))
        A[:, i] = np.concatenate([x, v])
    for i in range(P):
        x, v = step(np.zeros(P), np.zeros(P), np.eye(P)[i])
        B[:, i] = np.concatenate([x, v])
    return A, B, t


def test_harmonic_integrator_bias_is_small():
    """The exact stationary averages of the discrete step (a linear map with Gaussian noise: a discrete Lyapunov
    equation) differ from the exact finite-P value by less than _HARMONIC_BIAS_BOUND per degree of freedom (the largest
    difference, K_prim's, is 1.4e-4), less than one standard error of the sampled test below."""
    from scipy.linalg import solve_discrete_lyapunov

    P = _HO['P']
    A, B, t = _step_map(P, 1)
    S = solve_discrete_lyapunov(A, B @ B.T)
    xx = S[:P, :P]
    want = pimd_oracle.harmonic_value(P, _HO['kT'], _HO['hbar'], _HO['omega'])
    V = 0.5 * np.trace(xx) / P
    d = np.eye(P) - np.roll(np.eye(P), 1, axis=1)  # (x_j - x_j+1)
    K_prim = 0.5 * P * _HO['kT'] - t['kspring'] * np.trace(d @ xx @ d.T)
    cen = np.eye(P) - np.full((P, P), 1.0 / P)
    K_cv = 0.5 * _HO['kT'] + t['kvir'] * np.trace(cen @ xx)  # F = -x
    print('per degree of freedom: exact %.6f, step V %.6f K_prim %.6f K_cv %.6f' % (want, V, K_prim, K_cv))
    for got in (V, K_prim, K_cv):
        assert abs(got - want) < _HARMONIC_BIAS_BOUND
    assert want > 1.5 * 0.5 * _HO['kT']  # visibly quantum


_HARMONIC_BIAS_BOUND = 2.5e-4


def test_harmonic_quantum_statistics():
    """<V> (bead average), <K_prim> and <K_cv> of the restatement on an analytic harmonic force equal the exact
    finite-P value within 5 standard errors (block averages over the run; the seed is fixed), and sit well above the
    classical 3 kT / 2."""
    c = _HO
    P, n_poly, dimi = c['P'], 128, 3
    want = dimi * pimd_oracle.harmonic_value(P, c['kT'], c['hbar'], c['omega'])
    R0 = np.zeros((n_poly, P, dimi))
    V0 = np.zeros((n_poly, P, dimi))
    s = np.ones(dimi)
    args = (c['dt'], c['kT'], c['hbar'], c['gamma'], c['lam'])
    (R, V, F, E), _ = pimd_oracle.run(_harmonic, R0, V0, s, 400, *args, seed=17)
    _, fr = pimd_oracle.run(_harmonic, R, V, s, 2000, *args, seed=17, step0=400, stride=10, F=F, E=E)
    series = {'V': fr['E_pot'].mean((1, 2)), 'K_prim': fr['K_prim'].mean(1), 'K_cv': fr['K_cv'].mean(1)}
    for k, x in series.items():
        blocks = x.reshape(20, -1).mean(1)
        se = blocks.std(ddof=1) / np.sqrt(len(blocks))
        print('<%s> = %.5f, exact %.5f, standard error %.2g' % (k, x.mean(), want, se))
        assert abs(x.mean() - want) < 5.0 * se
        assert dimi * _HARMONIC_BIAS_BOUND < se  # the integrator's bias is below the resolution
    assert want > 1.5 * 0.5 * dimi * c['kT']


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_path_integral_dynamics_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLPathIntegralDynamics({'type': 'm'}, np.ones(3), n_beads=8)
    rc = _lib.lib().sgdml_b200_pimd_create(ctypes.byref(ctypes.c_void_p()), None, 1, 8, np.ones(3).ctypes.data)
    assert rc == -1002  # SGDML_B200_ERR_NO_DEVICE


def test_pimd_entry_points_and_constants():
    from sgdml_b200 import _lib, md

    for name in ('sgdml_b200_pimd_create', 'sgdml_b200_pimd_run'):
        assert name in _lib.SIGNATURES
    assert abs(md.HBAR_EV_FS - 0.6582119514) < 1e-10  # CODATA 2014, ASE's default
