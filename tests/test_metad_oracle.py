"""CPU checks of the metadynamics restatement (tests/metad_oracle.py) that the device tests compare against: the CV
gradients, the bias force's invariances, the deposition schedule, the reduction to plain MD, the walker and group
rules, and the well-tempered free-energy estimate of a diatomic double well against its exact profile."""

import numpy as np
import pytest

import md_oracle
import metad_oracle as mo

CVS = [('distance', (0, 1)), ('angle', (0, 1, 2)), ('dihedral', (0, 1, 2, 3)), ('dihedral', (3, 2, 1, 4))]


def _geoms(n, seed=0):
    return np.random.default_rng(seed).standard_normal((n, 5, 3)) * 1.2


def _numgrad(kind, atoms, X, h=1e-6, wrap=False):
    g = np.zeros((X.shape[0], len(atoms), 3))
    for p, a in enumerate(atoms):
        for x in range(3):
            Xp, Xm = X.copy(), X.copy()
            Xp[:, a, x] += h
            Xm[:, a, x] -= h
            d = mo.cv_eval(kind, atoms, Xp)[0] - mo.cv_eval(kind, atoms, Xm)[0]
            g[:, p, x] = (mo.wrap(d) if wrap else d) / (2 * h)
    return g


@pytest.mark.parametrize('kind,atoms', CVS[:3])
def test_cv_gradients(kind, atoms):
    X = _geoms(64)
    s, g = mo.cv_eval(kind, atoms, X)
    num = _numgrad(kind, atoms, X, wrap=kind == 'dihedral')
    assert np.max(np.abs(g - num)) < 1e-6 * max(1.0, np.max(np.abs(g)))
    if kind == 'angle':
        assert np.all((s >= 0) & (s <= np.pi))
    if kind == 'dihedral':
        assert np.all((s > -np.pi) & (s <= np.pi))


def test_dihedral_near_pi_and_degenerate_cases():
    # a trans dihedral at phi = pi - 1e-3 and pi + 1e-3 (which reads as -pi + 1e-3): the gradient is smooth across
    X = np.zeros((2, 4, 3))
    for r, phi in enumerate([np.pi - 1e-3, np.pi + 1e-3]):
        X[r] = [[1.0, 1.0, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 1.5], [np.cos(phi), np.sin(phi), 1.5]]
        X[r, 0] = [1.0, 0.0, 0.0]
    s, g = mo.cv_eval('dihedral', (0, 1, 2, 3), X)
    assert s[0] > 3.1 and s[1] < -3.1
    num = _numgrad('dihedral', (0, 1, 2, 3), X, wrap=True)
    assert np.max(np.abs(g - num)) < 1e-6
    assert np.max(np.abs(g[0] - g[1])) < 1e-2  # continuous through +-pi
    # collinear angle and dihedral with a collinear triple: defined zero gradients, no NaN
    Xc = np.array([[[0.0, 0, 0], [1.0, 0, 0], [2.0, 0, 0], [2.0, 1.0, 0]]])
    sa, ga = mo.cv_eval('angle', (0, 1, 2), Xc)
    sd, gd = mo.cv_eval('dihedral', (0, 1, 2, 3), Xc)
    assert sa[0] == np.pi and np.all(ga == 0) and np.all(gd == 0) and np.isfinite(sd[0])


def test_periodic_hill_difference():
    # a hill at +pi - 0.05 seen from -pi + 0.05 is 0.1 away, not 2 pi - 0.1; its dV/ds matches a central difference
    types = ['dihedral']
    C, W, H = np.array([[np.pi - 0.05]]), np.array([[0.2]]), np.array([1.0])
    V, dV = mo.hill_sum(np.array([-np.pi + 0.05]), types, C, W, H)
    assert abs(V - np.exp(-0.5 * (0.1 / 0.2) ** 2)) < 1e-12
    h = 1e-6
    num = (mo.hill_sum(np.array([-np.pi + 0.05 + h]), types, C, W, H)[0]
           - mo.hill_sum(np.array([-np.pi + 0.05 - h]), types, C, W, H)[0]) / (2 * h)
    assert abs(dV[0] - num) < 1e-7 and dV[0] < 0  # s lies 0.1 past the hill across the cut
    assert np.all(mo.wrap([np.pi, -np.pi, 2 * np.pi - 0.1]) < np.pi)


@pytest.mark.parametrize('j', range(4))
def test_bias_force_has_no_net_force_or_torque(j):
    X = _geoms(32, 1)
    R = X.reshape(32, -1)
    rng = np.random.default_rng(3)
    cvs = [CVS[j]]
    s0 = mo.bias(R, cvs, 32, [(np.zeros((0, 1)),) * 2 + (np.zeros(0),)])[0]
    hills = [(s0[:8] + 0.1 * rng.standard_normal((8, 1)), np.full((8, 1), 0.3), rng.uniform(0.5, 1.0, 8))]
    _, Vb, Fb, _ = mo.bias(R, cvs, 32, hills)
    F = Fb.reshape(32, 5, 3)
    scale = np.abs(F).max(axis=(1, 2))
    assert np.all(scale > 0)
    assert np.max(np.abs(F.sum(1)) / scale[:, None]) < 1e-13
    torque = np.cross(X, F).sum(1)
    assert np.max(np.abs(torque) / (scale * np.abs(X).max())[:, None]) < 1e-13


def _harmonic(k=1.0):
    def forces(R):
        X = R.reshape(R.shape[0], -1, 3)
        return 0.5 * k * (X * X).sum((1, 2)), -k * R

    return forces


def _setup(n_rep=4, seed=0):
    rng = np.random.default_rng(seed)
    R = _geoms(n_rep, seed).reshape(n_rep, -1)
    V = 0.1 * rng.standard_normal(R.shape)
    s = np.repeat(1.0 / np.linspace(1.0, 2.0, 5), 3)
    return R, V, s


def test_zero_height_is_plain_md_bit_for_bit():
    R, V, s = _setup()
    kw = dict(dt=0.01, gamma=0.5, kT=0.3, seed=11, step0=5, stride=5)
    fin, fr = mo.run(_harmonic(), R, V, s, CVS, 2, mo.empty_hills(2, 4), 40, w0=0.0, widths=np.full(4, 0.2), pace=3,
                     **kw)
    ref_fin, ref = md_oracle.run(_harmonic(), R, V, s, 40, **kw)
    for k in ref:
        assert np.array_equal(fr[k], ref[k]), k
    assert all(np.array_equal(a, b) for a, b in zip(fin[:4], ref_fin))
    assert all(len(g[2]) == 2 * mo.n_deposits(5, 40, 3) for g in fin[6])
    assert all(np.all(g[2] == 0.0) for g in fin[6])


def test_schedule_and_continuation():
    R, V, s = _setup()
    args = dict(dt=0.01, gamma=0.5, kT=0.3, w0=0.05, widths=np.array([0.1, 0.2, 0.3, 0.3]), pace=4, dkT=1.2, seed=3)
    hills0 = mo.empty_hills(2, 4)
    # the run's first state (step 8, a multiple of pace) deposits nothing: 8 steps from 8 deposit on 12 and 16
    fin, fr = mo.run(_harmonic(), R, V, s, CVS, 2, hills0, 8, step0=8, stride=1, **args)
    assert [len(g[2]) for g in fin[6]] == [4, 4]
    # the first hills were deposited at state 12 with the bias of state 12 (zero: nothing before it), heights w0
    assert np.all(fin[6][0][2][:2] == 0.05)
    assert np.array_equal(fin[6][0][0][:2], fr['cv'][3][:2])
    # the hills of state 12 bias state 13 onwards, not state 12
    assert np.all(fr['bias'][:4] == 0.0) and np.all(fr['bias'][4] > 0.0)
    # heights w0 exp(-V / dkT) of the depositing state's V
    assert np.allclose(fin[6][1][2][2:], 0.05 * np.exp(-fr['bias'][7][2:] / 1.2), rtol=0, atol=1e-16)
    # 2n steps are two runs of n steps, bit for bit
    fa, fra = mo.run(_harmonic(), R, V, s, CVS, 2, hills0, 5, step0=8, stride=1, **args)
    fb, frb = mo.run(_harmonic(), fa[0], fa[1], s, CVS, 2, fa[6], 3, step0=13, stride=1, **args)
    for k in fr:
        assert np.array_equal(fr[k], np.concatenate([fra[k], frb[k]])), k
    for g, h in zip(fin[6], fb[6]):
        assert all(np.array_equal(a, b) for a, b in zip(g, h))


def test_walkers_and_groups():
    R, V, s = _setup(6)
    args = dict(dt=0.01, gamma=0.5, kT=0.3, w0=0.05, widths=np.full(4, 0.2), pace=2, seed=3, stride=1)
    fin, fr = mo.run(_harmonic(), R, V, s, CVS, 3, mo.empty_hills(2, 4), 6, **args)
    assert [len(g[2]) for g in fin[6]] == [9, 9]  # 3 walkers x 3 deposits per group
    # each deposit holds the walkers' CVs in walker order
    assert np.array_equal(fin[6][1][0][3:6], fr['cv'][3][3:6])
    # groups are isolated: group 0 alone (first 3 replicas, with other noise streams for group 1) is unchanged
    R2 = R.copy()
    R2[3:] += 0.3
    fin2, fr2 = mo.run(_harmonic(), R2, V, s, CVS, 3, mo.empty_hills(2, 4), 6, **args)
    assert np.array_equal(fr2['R'][:, :3], fr['R'][:, :3]) and np.array_equal(fr2['bias'][:, :3], fr['bias'][:, :3])
    assert not np.array_equal(fr2['R'][:, 3:], fr['R'][:, 3:])
    assert all(np.array_equal(a, b) for a, b in zip(fin2[6][0], fin[6][0]))


# diatomic double well: U(d) = H ((d - d0)^2 - w^2)^2 / w^4, wells at d0 -+ w, the barrier H at d0; kT = 1
_D0, _W, _H = 1.5, 0.3, 4.0


def _dw(R):
    X = R.reshape(R.shape[0], 2, 3)
    r = X[:, 1] - X[:, 0]
    d = np.sqrt((r * r).sum(-1))
    y = (d - _D0) ** 2 - _W ** 2
    E = _H * y * y / _W ** 4
    dU = 4.0 * _H * y * (d - _D0) / _W ** 4
    f1 = -(dU / d)[:, None] * r
    return E, np.concatenate([-f1, f1], 1)


def test_well_tempered_profile_of_a_double_well():
    """The well-tempered estimate -gamma/(gamma-1) V(d) converges to the free energy U(d) - 2 kT ln d of the bond
    length (the Jacobian d^2).  Between the wells (d = 1.2 and 1.8) the ln term is 2 ln 1.5 = 0.81 kT and the barrier is
    4 kT, so the tolerance of 0.25 kT on the centred profile over [1.15, 1.85] fails for gamma in place of
    gamma/(gamma-1) (the profile scaled by 9) and for a profile without the ln term."""
    n_groups, n_walk = 1, 32
    n_rep = n_groups * n_walk
    R = np.zeros((n_rep, 6))
    R[:, 3] = np.where(np.arange(n_rep) % 2 == 0, _D0 - _W, _D0 + _W)
    s = np.ones(6)
    gamma_bf, kT = 10.0, 1.0
    fin, _ = mo.run(lambda x: _dw(x), R, np.zeros_like(R), s, [('distance', (0, 1))], n_walk,
                    mo.empty_hills(n_groups, 1), 6000, dt=0.02, gamma=1.0, kT=kT, w0=0.2, widths=[0.05], pace=40,
                    dkT=(gamma_bf - 1) * kT, seed=7)
    C, W, H = fin[6][0]
    d = np.linspace(1.15, 1.85, 29)
    Vb = (H[None] * np.exp(-0.5 * ((d[:, None] - C[None, :, 0]) / W[None, :, 0]) ** 2)).sum(1)
    y = (d - _D0) ** 2 - _W ** 2
    exact = _H * y * y / _W ** 4 - 2 * kT * np.log(d)

    def dev(f):
        f = f - f.mean()
        return np.max(np.abs(f - (exact - exact.mean())))

    est = -gamma_bf / (gamma_bf - 1) * Vb
    print('deviation %.3f kT; with gamma %.3f; without the ln term %.3f'
          % (dev(est), dev(-gamma_bf * Vb), np.max(np.abs((est - est.mean()) - (exact + 2 * kT * np.log(d))
                                                            + (exact + 2 * kT * np.log(d)).mean()))))
    assert dev(est) < 0.25
    assert dev(-gamma_bf * Vb) > 0.25
    no_ln = _H * y * y / _W ** 4
    assert np.max(np.abs((est - est.mean()) - (no_ln - no_ln.mean()))) > 0.25
