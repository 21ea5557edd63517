"""The NumPy restatement of the device nudged elastic band (tests/neb_oracle.py) on hand-built bands and on the
Mueller-Brown surface, and the CPU side of sgdml_b200_neb_fire / sgdml_b200.GDMLNEB: every tangent branch, the spring
and climbing forces, coincident images, a CI-NEB that finds the Mueller-Brown saddle located independently by a root
finder, linear interpolation with Kabsch alignment, the bound entry point and the loud failure without a device.
"""

import os
import types

import numpy as np
import pytest

import neb_oracle


def _band(t_minus, t_plus, E, F1, k=0.0, climb=False):
    """One band of three images of two atoms: R1 - R0 = t_minus, R2 - R1 = t_plus, model force F1 on the middle image
    -> its NEB force (6,)."""
    R = np.zeros((3, 6))
    R[1] = R[0] + np.asarray(t_minus, dtype=np.float64)
    R[2] = R[1] + np.asarray(t_plus, dtype=np.float64)
    F = np.zeros((3, 6))
    F[1] = F1
    Fn, top = neb_oracle.neb_force(R, F, np.asarray(E, dtype=np.float64), 3, k, climb)
    assert top.tolist() == [1]
    return Fn[0]


_F1 = np.array([1.0, 0.0, 0.0, 0.0, 0.0, 1.0])


def test_tangent_uphill_and_downhill():
    """E[i+1] > E[i] > E[i-1]: tau = t+;  E[i+1] < E[i] < E[i-1]: tau = t-.  |t+| = 2 and |t-| = 2 keep th exact."""
    tp, tm = [1.0, 1.0, 1.0, 1.0, 0.0, 0.0], [2.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    up = _band(tm, tp, [0.0, 1.0, 2.0], _F1)  # th = (1, 1, 1, 1, 0, 0) / 2, F.th = 1/2
    assert up.tolist() == [0.75, -0.25, -0.25, -0.25, 0.0, 1.0]
    down = _band(tm, tp, [2.0, 1.0, 0.0], _F1)  # th = (1, 0, 0, 0, 0, 0), F.th = 1
    assert down.tolist() == [0.0, 0.0, 0.0, 0.0, 0.0, 1.0]


def test_tangent_at_extrema_weights_by_energy_differences():
    """A maximum or minimum at i: tau = t+ dmax + t- dmin if E[i+1] > E[i-1], else t+ dmin + t- dmax."""
    # E = (0, 2, 1): dmax = 2 on t+, dmin = 1 on t-: (1, 1, 0, 0) 2 + (0, 0, 2, 2) 1 = (2, 2, 2, 2), th = 1/2 each
    a = _band([0.0, 0.0, 2.0, 2.0, 0.0, 0.0], [1.0, 1.0, 0.0, 0.0, 0.0, 0.0], [0.0, 2.0, 1.0], _F1)
    assert a.tolist() == [0.75, -0.25, -0.25, -0.25, 0.0, 1.0]
    # the other weighting would give (1, 1, 4, 4): not parallel to (1, 1, 1, 1)
    wrong = _band([0.0, 0.0, 2.0, 2.0, 0.0, 0.0], [1.0, 1.0, 0.0, 0.0, 0.0, 0.0], [1.0, 2.0, 0.0], _F1)
    assert wrong.tolist() != a.tolist()
    # E = (1, 2, 0): E[i+1] < E[i-1], dmin = 1 on t+, dmax = 2 on t-: (2, 2, 0, 0) 1 + (0, 0, 1, 1) 2 = (2, 2, 2, 2)
    b = _band([0.0, 0.0, 1.0, 1.0, 0.0, 0.0], [2.0, 2.0, 0.0, 0.0, 0.0, 0.0], [1.0, 2.0, 0.0], _F1)
    assert b.tolist() == a.tolist()
    # a minimum at i takes the same rule: E = (1, 0, 2) -> dmax = 2 (t+ side), dmin = 1
    c = _band([0.0, 0.0, 2.0, 2.0, 0.0, 0.0], [1.0, 1.0, 0.0, 0.0, 0.0, 0.0], [1.0, 0.0, 2.0], _F1)
    assert c.tolist() == a.tolist()


def test_coincident_images_give_no_nan():
    """|tau| = 0: th = 0, so the NEB force is the model force (and the spring term vanishes with it)."""
    for E in ([0.0, 1.0, 2.0], [0.0, 2.0, 1.0], [1.0, 1.0, 1.0]):
        for climb in (False, True):
            out = _band(np.zeros(6), np.zeros(6), E, _F1, k=5.0, climb=climb)
            assert out.tolist() == _F1.tolist()


def test_spring_term():
    """k (|t+| - |t-|) along th: |t+| = 2, |t-| = 1, th = t+ / 2, k = 3 -> 1.5 on each of th's coordinates."""
    out = _band([0.0, 0.0, 0.0, 0.0, 1.0, 0.0], [1.0, 1.0, 1.0, 1.0, 0.0, 0.0], [0.0, 1.0, 2.0], np.zeros(6), k=3.0)
    assert out.tolist() == [1.5, 1.5, 1.5, 1.5, 0.0, 0.0]


def test_climbing_image_reverses_the_tangent_force_without_spring():
    tp, tm = [1.0, 1.0, 1.0, 1.0, 0.0, 0.0], [2.0, 0.0, 0.0, 0.0, 0.0, 0.0]
    plain = _band(tm, tp, [0.0, 1.0, 2.0], _F1, k=0.0)
    climbing = _band(tm, tp, [0.0, 1.0, 2.0], _F1, k=3.0, climb=True)  # F - 2 (F.th) th, k ignored
    assert climbing.tolist() == [0.5, -0.5, -0.5, -0.5, 0.0, 1.0]
    assert (climbing - _F1).tolist() == (2.0 * (plain - _F1)).tolist()


def test_climbing_index_is_the_first_highest_interior_image():
    E = np.array([[9.0, 1.0, 5.0, 5.0, 2.0, 9.0], [0.0, 3.0, 3.0, 1.0, 3.0, 0.0], [0.0, np.nan, 1.0, 2.0, 0.0, 5.0]])
    # a NaN at image 1 compares false with everything, as in the kernel's scan: image 1 stays
    assert neb_oracle.climbing_index(E).tolist() == [2, 1, 1]


# --------------------------------------------------------------------------------- Mueller-Brown
_MB_A = np.array([-200.0, -100.0, -170.0, 15.0])
_MB_a = np.array([-1.0, -1.0, -6.5, 0.7])
_MB_b = np.array([0.0, 0.0, 11.0, 0.6])
_MB_c = np.array([-10.0, -10.0, -6.5, 0.7])
_MB_x0 = np.array([1.0, 0.0, -0.5, -1.0])
_MB_y0 = np.array([0.0, 0.5, 1.5, 1.0])


def _mb_terms(p):
    p = np.asarray(p, dtype=np.float64)
    dx, dy = p[..., 0:1] - _MB_x0, p[..., 1:2] - _MB_y0
    return dx, dy, _MB_A * np.exp(_MB_a * dx * dx + _MB_b * dx * dy + _MB_c * dy * dy)


def _mb(p):
    return _mb_terms(p)[2].sum(-1)


def _mb_grad(p):
    dx, dy, e = _mb_terms(p)
    return np.stack([(e * (2 * _MB_a * dx + _MB_b * dy)).sum(-1), (e * (_MB_b * dx + 2 * _MB_c * dy)).sum(-1)], -1)


def _mb_hess(p):
    dx, dy, e = _mb_terms(p)
    gx, gy = 2 * _MB_a * dx + _MB_b * dy, _MB_b * dx + 2 * _MB_c * dy
    hxy = (e * (gx * gy + _MB_b)).sum(-1)
    return np.array([[(e * (gx * gx + 2 * _MB_a)).sum(-1), hxy], [hxy, (e * (gy * gy + 2 * _MB_c)).sum(-1)]])


def _mb_forces(R):
    """Mueller-Brown in the (x, y) pair of a one-atom system; z feels no force."""
    F = np.zeros_like(R)
    F[:, :2] = -_mb_grad(R[:, :2])
    return _mb(R[:, :2]), F


def test_ci_neb_finds_the_mueller_brown_saddle():
    """The saddle between the minima near (-0.558, 1.442) and (-0.050, 0.467), found by a root finder on grad V = 0 from
    the literature point (-0.822, 0.624), is a first-order saddle; a CI-NEB of the restatement between the two minima
    puts its climbing image there."""
    import scipy.optimize as so

    mA = so.minimize(_mb, [-0.558, 1.442], jac=_mb_grad, tol=1e-12).x
    mB = so.minimize(_mb, [-0.050, 0.467], jac=_mb_grad, tol=1e-12).x
    sad = so.root(_mb_grad, [-0.822, 0.624], jac=_mb_hess, tol=1e-12).x
    assert np.max(np.abs(_mb_grad(sad))) < 1e-9
    ev = np.linalg.eigvalsh(_mb_hess(sad))
    assert (ev < 0).sum() == 1, ev
    assert np.allclose(sad, [-0.822, 0.624], atol=2e-3)

    P = 9
    R = np.zeros((P, 3))
    R[:, :2] = mA + np.linspace(0.0, 1.0, P)[:, None] * (mB - mA)
    dt, maxstep, k = 0.002, 0.05, 10.0
    plain = neb_oracle.neb_fire(_mb_forces, R, P, 3000, 1e-2, k, False, maxstep, dt, 10 * dt)
    assert plain['converged'].all()
    ci = neb_oracle.neb_fire(_mb_forces, plain['R'], P, 20000, 1e-3, k, True, maxstep, dt, 10 * dt)
    assert ci['converged'].all() and ci['fmax'][0] < 1e-3
    top = int(ci['climbing'][0])
    x = ci['R'][top, :2]
    print('climbing image %d at %s, saddle %s, %d + %d steps' % (top, x, sad, plain['n_steps'][0], ci['n_steps'][0]))
    assert np.max(np.abs(x - sad)) < 1e-3
    assert abs(_mb(x) / _mb(sad) - 1.0) < 1e-3
    # the endpoints never moved
    assert np.array_equal(ci['R'][[0, P - 1]], R[[0, P - 1]])


def test_band_fire_is_one_vector_per_band():
    """Two bands in one call equal each band alone: the band sums never mix bands."""
    P = 5
    rng = np.random.default_rng(0)
    R = np.zeros((2 * P, 3))
    for b, (a, z) in enumerate([((-0.558, 1.442), (-0.050, 0.467)), ((0.623, 0.028), (-0.050, 0.467))]):
        R[b * P:(b + 1) * P, :2] = np.array(a) + np.linspace(0.0, 1.0, P)[:, None] * (np.array(z) - np.array(a))
    R[:, :2] += 1e-2 * rng.standard_normal((2 * P, 2))
    both = neb_oracle.neb_fire(_mb_forces, R, P, 40, 0.0, 5.0, True, 0.05, 0.002, 0.02)
    for b in range(2):
        one = neb_oracle.neb_fire(_mb_forces, R[b * P:(b + 1) * P], P, 40, 0.0, 5.0, True, 0.05, 0.002, 0.02)
        assert np.array_equal(one['R'], both['R'][b * P:(b + 1) * P])
        assert one['fmax'][0] == both['fmax'][b] and one['climbing'][0] == both['climbing'][b]


# --------------------------------------------------------------------------------- interpolate
def _neb_stub(periodic=False, n_images=5):
    from sgdml_b200.md import GDMLNEB

    obj = GDMLNEB.__new__(GDMLNEB)
    obj.n_images = n_images
    obj.gdml_predict = types.SimpleNamespace(lat_and_inv=(np.eye(3), np.eye(3)) if periodic else None)
    return obj


def test_interpolate_reproduces_endpoints_and_aligns_rigid_copies():
    from scipy.spatial.transform import Rotation

    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 7, 3))
    y = rng.standard_normal((2, 7, 3))
    neb = _neb_stub()
    band = neb.interpolate(x, y, 6, align=False)
    assert band.shape == (2, 6, 7, 3)
    assert np.array_equal(band[:, 0], x) and np.array_equal(band[:, -1], y)
    assert np.allclose(band[:, 2], x + 0.4 * (y - x), rtol=0, atol=1e-15)
    # a rigidly rotated and translated copy aligns back onto the original: every image is the original
    Q = Rotation.random(2, random_state=4).as_matrix()
    moved = np.einsum('bij,baj->bai', Q, x) + np.array([[[1.5, -2.0, 0.25]], [[-3.0, 0.5, 7.0]]])
    aligned = neb.interpolate(x, moved, 4, align=True)
    assert np.array_equal(aligned[:, 0], x)
    assert np.max(np.abs(aligned - x[:, None])) < 1e-12
    # the default image count is the instance's
    assert neb.interpolate(x[0], y[0], align=False).shape == (5, 7, 3)


def test_interpolate_refuses_alignment_of_periodic_models():
    neb = _neb_stub(periodic=True)
    x = np.zeros((3, 3))
    with pytest.raises(ValueError, match='periodic'):
        neb.interpolate(x, x + 1.0, 5)
    assert neb.interpolate(x, x + 1.0, 5, align=False).shape == (5, 3, 3)


# --------------------------------------------------------------------------------- bindings
def test_neb_entry_point_is_bound():
    import ctypes

    import sgdml_b200
    from sgdml_b200 import _lib

    restype, args = _lib.SIGNATURES['sgdml_b200_neb_fire']
    assert restype is ctypes.c_int
    assert args == [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_double, ctypes.c_double, ctypes.c_int,
                    ctypes.c_double, ctypes.c_double, ctypes.c_double] + [ctypes.c_void_p] * 5
    getattr(_lib.lib(), 'sgdml_b200_neb_fire')
    assert sgdml_b200.GDMLNEB.neb and sgdml_b200.GDMLNEB.interpolate


def test_neb_has_no_md_run():
    from sgdml_b200.md import GDMLNEB

    with pytest.raises(TypeError, match='GDMLDynamics'):
        GDMLNEB.__new__(GDMLNEB).run(10, 0.5)


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_neb_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    import sgdml_b200
    from sgdml_b200 import _lib

    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        sgdml_b200.GDMLNEB({'type': 'm'}, 5)
    assert _lib.lib().sgdml_b200_neb_fire(None, 5, 10, 0.05, 0.1, 0, 0.2, 0.1, 1.0, None, None, None, None,
                                          None) == -1002
