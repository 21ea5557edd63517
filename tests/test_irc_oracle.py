"""The NumPy restatement of the device reaction path (tests/irc_oracle.py) on exact surfaces, and the CPU side of
sgdml_b200_irc_rk4 / sgdml_b200.GDMLIRC: on a quadratic bowl with unequal masses the RK4 points lie on the exact
steepest-descent path and converge at fourth order; on the Mueller-Brown surface the two branches from the saddle end
next to the two minima it connects and follow the path an accurate ODE solver gives; the three end codes; equal masses
give a mass-independent Cartesian path; the bound entry point and the loud failure without a device.
"""

import os

import numpy as np
import pytest

import irc_oracle
from test_neb_oracle import _mb, _mb_forces, _mb_grad, _mb_hess

_MB_SADDLE0 = (-0.822, 0.624)
_MB_MINIMA = ((-0.558, 1.442), (-0.050, 0.467))


def _bowl(A, r):
    """E = 1/2 x^T A x in the mass-weighted coordinates x = R / r of a 2-atom system: F = -(A x) / r."""
    def forces(R):
        x = R / r
        Ax = x @ A.T
        return 0.5 * np.einsum('bi,bi->b', x, Ax), -(Ax / r)
    return forces


def _bowl_setup():
    rng = np.random.default_rng(4)
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    A = Q @ np.diag([0.6, 0.9, 1.3, 1.8, 2.4, 3.0]) @ Q.T
    r = np.sqrt(1.0 / np.repeat([1.0, 4.0], 3))  # masses 1 and 4
    x1 = rng.standard_normal(6)
    return A, r, x1


def _bowl_path(A, r, x1, h, max_points):
    """The restatement started so that its point 1 is x1 for every h: saddle x1 - h v, v the descent direction at x1.
    Returns the forward branch's mass-weighted points 1, 2, ... (arc length (n - 1) h from x1)."""
    f = _bowl(A, r)
    v = -(A @ x1) / np.linalg.norm(A @ x1)
    R0 = (r * (x1 - h * v))[None]
    E0, F0 = f(R0)
    out = irc_oracle.irc(f, R0, E0, F0, (r * v)[None], r * r, max_points, h, 0.0)
    n = out['n_points'][0]
    return out['R_path'][0, 1:n] / r, out


def _bowl_exact(A, x1, S):
    """exp(-A t) x1 at arc length S from x1 (the arc length by quadrature, t by root finding)."""
    import scipy.integrate as si
    import scipy.optimize as so

    w, Q = np.linalg.eigh(A)
    y1 = Q.T @ x1
    x = lambda t: Q @ (np.exp(-w * t) * y1)  # noqa: E731
    speed = lambda t: np.linalg.norm(w * np.exp(-w * t) * y1)  # noqa: E731
    arc = lambda t: si.quad(speed, 0.0, t, epsabs=1e-13, epsrel=1e-13, limit=200)[0]  # noqa: E731
    t = so.brentq(lambda t: arc(t) - S, 0.0, 50.0, xtol=1e-15, rtol=1e-15)
    return x(t)


def test_quadratic_bowl_points_lie_on_the_exact_path_at_fourth_order():
    """With unequal masses the exact mass-weighted path from x1 is exp(-A t) x1; the RK4 points at arc length (n - 1) h
    lie on it, and at a fixed arc length the error for h against h / 2 falls by 12 to 20 (fourth order: 16)."""
    A, r, x1 = _bowl_setup()
    S = 0.8
    errs = []
    for h in (0.1, 0.05):
        pts, out = _bowl_path(A, r, x1, h, int(round(S / h)) + 2)
        assert out['end'][0] == 3  # still descending at S
        assert np.all(np.diff(out['E_path'][0, :out['n_points'][0]]) < 0.0)
        for n in range(0, len(pts), 4):
            assert np.linalg.norm(pts[n] - _bowl_exact(A, x1, n * h)) < 1e-4
        errs.append(np.linalg.norm(pts[int(round(S / h))] - _bowl_exact(A, x1, S)))
    ratio = errs[0] / errs[1]
    print('bowl: errors at s = %.2f: %.3e (h), %.3e (h / 2), ratio %.2f' % (S, errs[0], errs[1], ratio))
    assert 12.0 < ratio < 20.0


def _mb_saddle():
    import scipy.optimize as so

    sad = so.root(lambda p: _mb_grad(p), _MB_SADDLE0, tol=1e-14).x
    w, U = np.linalg.eigh(_mb_hess(sad))
    assert w[0] < 0.0 < w[1]
    return sad, U[:, 0]


def _mb_irc(h, max_points=2000, fmax=1.0):
    sad, u = _mb_saddle()
    R0 = np.array([[sad[0], sad[1], 0.0]])
    E0, F0 = _mb_forces(R0)
    mode = np.array([[u[0], u[1], 0.0]])
    return irc_oracle.irc(_mb_forces, R0, E0, F0, mode, np.ones(3), max_points, h, fmax), sad, u


def test_mueller_brown_branches_reach_both_minima():
    """From the saddle near (-0.822, 0.624) along its Hessian's negative eigenvector, one branch ends next to the
    minimum near (-0.558, 1.442) and the other next to the one near (-0.050, 0.467); a minimiser from each end lands on
    that minimum; the energies fall strictly along both branches."""
    import scipy.optimize as so

    out, sad, u = _mb_irc(0.01)
    mins = [so.minimize(_mb, m, jac=_mb_grad, method='BFGS', options={'gtol': 1e-10}).x for m in _MB_MINIMA]
    ends = out['R'][:, :2]
    print('Mueller-Brown: points %s, end codes %s, ends %s' % (out['n_points'].tolist(), out['end'].tolist(),
                                                              ends.tolist()))
    hit = []
    for b in range(2):
        n = out['n_points'][b]
        assert out['end'][b] in (1, 2) and n > 10
        assert np.all(np.diff(out['E_path'][b, :n]) < 0.0)
        assert np.all(np.isnan(out['E_path'][b, n:])) and np.all(np.isnan(out['R_path'][b, n:]))
        d = [np.linalg.norm(ends[b] - m) for m in mins]
        k = int(np.argmin(d))
        assert d[k] < 0.02, d
        m = so.minimize(_mb, ends[b], jac=_mb_grad, method='BFGS', options={'gtol': 1e-10}).x
        assert np.linalg.norm(m - mins[k]) < 1e-6
        hit.append(k)
    assert sorted(hit) == [0, 1]


def test_mueller_brown_path_follows_the_ode_solution():
    """The RK4 points at arc length (n - 1) h from point 1 agree with solve_ivp (rtol 1e-12) of the same normalised
    flow dx/ds = -grad E / |grad E| to 5e-6 (RK4's global error at h = 0.01 is about 1e-6), until |grad E| falls
    below 10 on the way into the minimum, where the flow turns sharply."""
    import scipy.integrate as si

    h = 0.01
    out, sad, u = _mb_irc(h)
    flow = lambda s, p: -_mb_grad(p) / np.linalg.norm(_mb_grad(p))  # noqa: E731
    worst = 0.0
    for b in range(2):
        n = out['n_points'][b]
        P = out['R_path'][b, 1:n, :2]
        g = np.linalg.norm(_mb_grad(P), axis=1)
        top = int(np.argmax(g))
        keep = np.arange(top + int(np.argmax(g[top:] < 10.0)))  # up to the first small gradient past the steepest
        S = h * keep
        sol = si.solve_ivp(flow, (0.0, S[-1]), P[0], method='DOP853', rtol=1e-12, atol=1e-12, t_eval=S)
        err = np.max(np.linalg.norm(sol.y.T - P[keep], axis=1))
        worst = max(worst, err)
        assert len(keep) > 20
    print('Mueller-Brown: largest distance from the ODE solution %.3e' % worst)
    assert worst < 5e-6


def test_end_codes():
    """A start at the bowl's minimum rises both ways: end 2 at point 0, the state back on the start.  max_points = 2:
    end 3 after point 1.  A large fmax: end 1 at point 1."""
    A, r, _ = _bowl_setup()
    f = _bowl(A, r)
    R0 = np.zeros((1, 6))
    E0, F0 = f(R0)
    out = irc_oracle.irc(f, R0, E0, F0, np.ones((1, 6)), r * r, 10, 0.05, 0.0)
    assert np.array_equal(out['end'], [2, 2]) and np.array_equal(out['n_points'], [1, 1])
    assert np.all(out['R'] == 0.0) and np.all(out['E'] == 0.0) and np.all(out['fmax'] == 0.0)
    assert np.all(np.isnan(out['R_path'][:, 1:])) and np.all(out['E_path'][:, 0] == 0.0)
    two, _, _ = _mb_irc(0.01, max_points=2, fmax=0.0)
    assert np.array_equal(two['end'], [3, 3]) and np.array_equal(two['n_points'], [2, 2])
    assert np.array_equal(two['R'], two['R_path'][:, 1])
    big, _, _ = _mb_irc(0.01, fmax=1e6)
    assert np.array_equal(big['end'], [1, 1]) and np.array_equal(big['n_points'], [2, 2])
    assert np.all(big['fmax'] < 1e6)
    with pytest.raises(ValueError):
        irc_oracle.irc(f, R0, E0, F0, np.zeros((1, 6)), r * r, 10, 0.05, 0.0)
    with pytest.raises(ValueError):
        irc_oracle.irc(f, R0, E0, F0, np.full((1, 6), np.nan), r * r, 10, 0.05, 0.0)


def test_equal_masses_give_a_mass_independent_path():
    """All masses m: the Cartesian path with step h sqrt(m) does not depend on m, and its mass-weighted arc length
    scales as sqrt(m)."""
    sad, u = _mb_saddle()
    R0 = np.array([[sad[0], sad[1], 0.0]])
    E0, F0 = _mb_forces(R0)
    mode = np.array([[u[0], u[1], 0.0]])
    runs = []
    for m in (1.0, 4.0, 12.0):
        runs.append(irc_oracle.irc(_mb_forces, R0, E0, F0, mode, np.full(3, 1.0 / m), 300, 0.01 * np.sqrt(m), 1.0))
    for m, o in zip((4.0, 12.0), runs[1:]):
        assert np.array_equal(o['n_points'], runs[0]['n_points']) and np.array_equal(o['end'], runs[0]['end'])
        assert np.nanmax(np.abs(o['R_path'] - runs[0]['R_path'])) < 1e-12
        for b in range(2):
            n = o['n_points'][b]
            arc = lambda P, mm: np.linalg.norm(np.diff(P * np.sqrt(mm), axis=0), axis=1).sum()  # noqa: E731
            ratio = arc(o['R_path'][b, :n], m) / arc(runs[0]['R_path'][b, :n], 1.0)
            assert abs(ratio / np.sqrt(m) - 1.0) < 1e-12


# --------------------------------------------------------------------------------- bindings
def test_irc_entry_point_is_bound():
    import ctypes

    import sgdml_b200
    from sgdml_b200 import _lib

    restype, args = _lib.SIGNATURES['sgdml_b200_irc_rk4']
    assert restype is ctypes.c_int
    assert args == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_double] * 2 + [ctypes.c_void_p] * 6
    getattr(_lib.lib(), 'sgdml_b200_irc_rk4')
    assert sgdml_b200.GDMLIRC.run


def test_modes_must_be_float64_cuda_tensors():
    """Torch saddles and modes that are not float64 CUDA tensors are refused before anything reaches the engine (the
    entry point reads n_saddles 3N doubles from the pointer)."""
    import torch

    from sgdml_b200.md import GDMLIRC

    obj = GDMLIRC.__new__(GDMLIRC)
    obj.n_saddles, obj.n_atoms, obj.n_replicas = 2, 3, 4
    for x in (torch.zeros(2, 3, 3), torch.zeros(2, 3, 3, dtype=torch.float64), torch.zeros(2, 3, 3, dtype=torch.int64)):
        with pytest.raises(ValueError, match='float64 CUDA'):
            obj.run(x, np.zeros((2, 3, 3)))
        with pytest.raises(ValueError, match='float64 CUDA'):
            obj.run(np.zeros((2, 3, 3)), x)
        with pytest.raises(ValueError, match='float64 CUDA'):
            obj._irc_raw(x.reshape(2, 9), 10, 0.05, 0.0)
    with pytest.raises(ValueError, match=r'\(n_saddles, 3N\)'):
        obj._irc_raw(np.zeros((2, 8)), 10, 0.05, 0.0)
    with pytest.raises(ValueError, match='n_saddles'):
        obj.run(np.zeros((3, 3, 3)), np.zeros((3, 3)))
    with pytest.raises(ValueError, match='step'):
        obj.run(np.zeros((3, 3)), np.ones((3, 3)), step=0.0)


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_irc_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLIRC({'type': 'm'}, np.ones(3), 2)
    assert _lib.lib().sgdml_b200_irc_rk4(None, None, 10, 0.05, 0.05, None, None, None, None, None, None) == -1002
