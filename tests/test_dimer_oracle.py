"""The NumPy restatement of the device dimer search (tests/dimer_oracle.py) on exact quadratics and on the Mueller-Brown
surface, and the CPU side of sgdml_b200_dimer_fire / sgdml_b200.GDMLDimer: one rotation finds the lowest eigenvector of
a quadratic in both half-angle branches, the rigid projection removes translations and rotations (and only
translations for a linear molecule's rotations it cannot define), a search from a Mueller-Brown minimum ends on a
first-order saddle located independently by a root finder, the bound entry point and the loud failure without a
device.
"""

import os

import numpy as np
import pytest

import dimer_oracle
from test_neb_oracle import _mb, _mb_forces, _mb_grad, _mb_hess

_PHI = np.pi / 4


def _quadratic(A):
    """E = 1/2 x^T A x in the (x, y) pair of a one-atom system; z feels no force."""
    def forces(R):
        F = np.zeros_like(R)
        F[:, :2] = -(R[:, :2] @ A.T)
        return 0.5 * np.einsum('bi,ij,bj->b', R[:, :2], A, R[:, :2]), F
    return forces


def _one_rotation(A, n0, x0=(0.3, -0.7)):
    R = np.zeros((2, 3))
    R[0, :2] = x0
    mode = np.array([[n0[0], n0[1], 0.0]])
    # two replays: the trial rotation, then the fit, the rotation and one translation
    return dimer_oracle.search(_quadratic(A), R, mode, 2, 0.0, 1e-4, np.cos(_PHI), np.sin(_PHI), 0.0, 0.1, 0.01, 0.1,
                               project_='none')


@pytest.mark.parametrize('angle', [0.3, 0.7, 1.2, 1.45, 2.6])
def test_one_rotation_finds_the_lowest_eigenvector_of_a_quadratic(angle):
    """On E = 1/2 x^T A x with one negative eigenvalue, the fitted C(phi) is exact, so one rotation turns any start
    mode onto the lowest eigenvector and C_use is its eigenvalue.  Starts within 45 degrees of it take the c2 >= 0
    branch of the half angle, the others the c2 < 0 branch."""
    Q = np.array([[np.cos(0.4), -np.sin(0.4)], [np.sin(0.4), np.cos(0.4)]])
    lam = np.array([-3.0, 5.0])
    A = Q @ np.diag(lam) @ Q.T
    vmin = Q[:, 0]
    start = np.array([np.cos(0.4 + angle), np.sin(0.4 + angle)])  # `angle` radians from vmin
    out = _one_rotation(A, start)
    assert out['n_rot'][0] == 1 and out['n_steps'][0] == 1
    n = out['modes'][0]
    assert n[2] == 0.0
    assert abs(abs(n[:2] @ vmin) - 1.0) < 1e-9 and np.linalg.norm(n) == pytest.approx(1.0, abs=1e-15)
    assert abs(out['C_use'][0] / lam[0] - 1.0) < 1e-9
    assert abs(out['curvature'][0] / lam[0] - 1.0) < 1e-9  # measured again at the moved centre
    near = min(angle % np.pi, np.pi - angle % np.pi) < np.pi / 4
    assert (out['c2'][0] >= 0.0) == near


def test_convex_region_moves_up_the_mode():
    """Both eigenvalues positive: C_use > 0, and the translation force is -(F.N) N, uphill along the lowest mode."""
    A = np.diag([1.0, 4.0])
    out = _one_rotation(A, (np.cos(0.2), np.sin(0.2)), x0=(0.5, 0.0))
    assert out['C_use'][0] == pytest.approx(1.0, rel=1e-9)
    assert out['R'][0, 0] > 0.5 and abs(out['R'][0, 1]) < 1e-9  # away from the minimum along x


def _rigid_basis(r):
    x = r.reshape(-1, 3) - r.reshape(-1, 3).mean(0)
    out = []
    for k in range(3):
        t = np.zeros_like(x)
        t[:, k] = 1.0
        out.append(t.ravel())
        e = np.zeros(3)
        e[k] = 1.0
        out.append(np.cross(e, x).ravel())
    return [v / np.linalg.norm(v) for v in out]


def test_projection_removes_rigid_motions():
    rng = np.random.default_rng(4)
    r = rng.standard_normal(15) * 1.5 + 3.0
    n, _ = dimer_oracle.project(rng.standard_normal(15), r)
    assert abs(np.linalg.norm(n) - 1.0) < 1e-15
    for v in _rigid_basis(r):
        assert abs(n @ v) < 1e-13
    # translations only: the rotations stay
    t, _ = dimer_oracle.project(rng.standard_normal(15), r, 'translations')
    basis = _rigid_basis(r)
    assert all(abs(t @ basis[k]) < 1e-13 for k in (0, 2, 4))
    assert max(abs(t @ basis[k]) for k in (1, 3, 5)) > 1e-3


def test_rigid_modes_are_rejected():
    rng = np.random.default_rng(5)
    r = rng.standard_normal(12)
    for v in _rigid_basis(r):
        with pytest.raises(ValueError, match='rigid'):
            dimer_oracle.init_mode(3.0 * v, r)
    for bad in (np.zeros(12), np.full(12, np.nan), np.r_[np.inf, np.ones(11)]):
        with pytest.raises(ValueError):
            dimer_oracle.init_mode(bad, r)
    # a rotation is a fine mode when only the translations are removed
    n = dimer_oracle.init_mode(_rigid_basis(r)[1], r, 'translations')
    assert abs(abs(n @ _rigid_basis(r)[1]) - 1.0) < 1e-12


def test_linear_molecule_drops_the_rotational_part():
    """Atoms on a line: I is singular, det <= 1e-10 (tr I / 3)^3, so only the translations go (one atom likewise, but
    then nothing is left: test_rigid_modes_are_rejected)."""
    rng = np.random.default_rng(6)
    r = (np.linspace(-1.0, 2.0, 4)[:, None] * np.array([0.3, -0.5, 0.8])).ravel()
    src = rng.standard_normal(12)
    a, _ = dimer_oracle.project(src, r)
    b, _ = dimer_oracle.project(src, r, 'translations')
    assert np.array_equal(a, b)


def test_search_finds_a_mueller_brown_saddle():
    """From the minimum near (-0.050, 0.467), nudged along a seeded mode, the search ends at a point where
    scipy.optimize.root moves less than 1e-3, the Hessian has exactly one negative eigenvalue, and the mode lies along
    its eigenvector."""
    import scipy.optimize as so

    m = so.minimize(_mb, [-0.050, 0.467], jac=_mb_grad, tol=1e-12).x
    rng = np.random.default_rng(11)
    R = np.zeros((2, 3))
    mode = np.zeros((1, 3))
    mode[0, :2] = rng.standard_normal(2)
    R[0, :2] = m + 0.01 * mode[0, :2] / np.linalg.norm(mode[0, :2])
    out = dimer_oracle.search(_mb_forces, R, mode, 4000, 1e-3, 1e-4, np.cos(_PHI), np.sin(_PHI), 0.1, 0.02, 1e-3,
                              1e-2, project_='none')
    x = out['R'][0, :2]
    assert out['converged'][0], (out['fmax'], out['n_steps'])
    sad = so.root(_mb_grad, x, jac=_mb_hess, tol=1e-12).x
    print('saddle %s after %d translations, %d rotations; root moved %.2e' % (
        x, out['n_steps'][0], out['n_rot'][0], np.max(np.abs(sad - x))))
    assert np.max(np.abs(sad - x)) < 1e-3
    ev, vec = np.linalg.eigh(_mb_hess(x))
    assert (ev < 0).sum() == 1, ev
    assert abs(out['modes'][0, :2] @ vec[:, 0]) > 0.999
    assert out['curvature'][0] < 0.0 and abs(out['curvature'][0] / ev[0] - 1.0) < 1e-2
    assert np.linalg.norm(sad - m) > 0.1  # not the minimum


def test_dimers_are_independent():
    """Two dimers in one call equal each alone: the sums never mix dimers."""
    A = np.array([[2.0, 1.0], [1.0, -1.0]])
    R = np.zeros((4, 3))
    R[0, :2], R[2, :2] = (0.3, 0.1), (-0.2, 0.5)
    modes = np.array([[1.0, 0.2, 0.0], [0.1, 1.0, 0.0]])
    args = (10, 1e-6, 1e-4, np.cos(_PHI), np.sin(_PHI), 0.0, 0.1, 0.01, 0.1)
    both = dimer_oracle.search(_quadratic(A), R, modes, *args, project_='none')
    for d in range(2):
        one = dimer_oracle.search(_quadratic(A), R[2 * d:2 * d + 2], modes[d:d + 1], *args, project_='none')
        assert np.array_equal(one['R'], both['R'][2 * d:2 * d + 2])
        assert one['curvature'][0] == both['curvature'][d] and one['n_rot'][0] == both['n_rot'][d]


def test_translation_fire_is_relax_oracle_fire():
    """The dimer's per-vector FIRE step (dimer_oracle._Fire, fire_update's restatement one step at a time) driven by a
    force function gives relax_oracle.fire's trajectory bit for bit, through mixing, growth of dt and resets."""
    import relax_oracle

    R0 = np.array([[0.55, 0.05, 0.0]])
    args = (0.05, 2e-3, 2e-2)  # maxstep, dt, dtmax: large enough on Mueller-Brown to overshoot and reset
    for steps in (1, 2, 40):
        ref = relax_oracle.fire(_mb_forces, R0, steps, 0.0, *args)
        fire = dimer_oracle._Fire()
        r, v = R0[0].copy(), np.zeros(3)
        resets = 0
        for _ in range(steps):
            F = _mb_forces(r[None])[1][0]
            fire.update(r, v, F, args[1], args[2], args[0])
            resets += fire.n_steps > 1 and fire.n_pos == 0
        assert np.array_equal(r, ref['R'][0]) and np.array_equal(v, ref['V'][0])
        assert (fire.dt, fire.alpha, fire.n_pos, fire.n_steps) == (ref['dt'][0], ref['alpha'][0], ref['n_pos'][0],
                                                                   ref['n_steps'][0])
    assert resets > 0 and ref['dt'][0] != args[1]  # both branches ran


def test_modes_must_be_float64_cuda_tensors():
    """Torch modes and positions that are not float64 CUDA tensors are refused before anything reaches the engine
    (the entry point reads n_dimers 3N doubles from the pointer)."""
    import torch

    from sgdml_b200.md import GDMLDimer

    obj = GDMLDimer.__new__(GDMLDimer)
    obj.n_dimers, obj.n_atoms = 2, 3
    for x in (torch.zeros(2, 3, 3), torch.zeros(2, 3, 3, dtype=torch.float64), torch.zeros(2, 3, 3, dtype=torch.int64)):
        for name in ('modes', 'positions'):
            with pytest.raises(ValueError, match='float64 CUDA'):
                obj._per_dimer(x, name)
        with pytest.raises(ValueError, match='float64 CUDA'):
            obj._dimer_raw(x.reshape(2, 9), 10, 0.0, 1e-4, _PHI, _PHI, 0.0, 0.1, 0.1, 1.0)
        with pytest.raises(ValueError, match='float64 CUDA'):
            obj.search(modes=x)
    with pytest.raises(ValueError, match=r'\(n_dimers, 3N\)'):
        obj._dimer_raw(np.zeros((2, 8)), 10, 0.0, 1e-4, _PHI, _PHI, 0.0, 0.1, 0.1, 1.0)


# --------------------------------------------------------------------------------- bindings
def test_dimer_entry_point_is_bound():
    import ctypes

    import sgdml_b200
    from sgdml_b200 import _lib

    restype, args = _lib.SIGNATURES['sgdml_b200_dimer_fire']
    assert restype is ctypes.c_int
    assert args == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_double] * 8 + [ctypes.c_void_p] * 7
    getattr(_lib.lib(), 'sgdml_b200_dimer_fire')
    assert sgdml_b200.GDMLDimer.search


def test_dimer_has_no_md_run():
    from sgdml_b200.md import GDMLDimer

    with pytest.raises(TypeError, match='GDMLDynamics'):
        GDMLDimer.__new__(GDMLDimer).run(10, 0.5)


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_dimer_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLDimer({'type': 'm'}, 4).search(np.zeros((3, 3)))
    assert _lib.lib().sgdml_b200_dimer_fire(None, None, 10, 0.05, 1e-4, 0.7071067811865476, 0.7071067811865476, 0.1,
                                            0.2, 0.1, 1.0, None, None, None, None, None, None, None) == -1002
