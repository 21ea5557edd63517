"""The NumPy restatement of the vibrational analysis (tests/vib_oracle.py) and the host-side thermochemistry and rate of
sgdml_b200.vib against closed forms: a diatomic spring, a spring network against the eigenvalues of its
central-difference Hessian, rigid-mode counts, invariance under rigid motions, the thermo limits and Vineyard's rate on
a separable quadratic saddle."""

import math

import numpy as np
import pytest

import vib_oracle as vo


def _springs(X, pairs, k, d0):
    """Energy and forces (eV, eV / Angstrom) of harmonic springs 0.5 k (d - d0)^2 on `pairs`."""
    X = X.reshape(-1, 3)
    E, F = 0.0, np.zeros_like(X)
    for (a, b), kk, dd in zip(pairs, k, d0):
        v = X[a] - X[b]
        d = np.linalg.norm(v)
        E += 0.5 * kk * (d - dd) ** 2
        f = -kk * (d - dd) * v / d
        F[a] += f
        F[b] -= f
    return E, F.ravel()


def _fd_hessian(X, pairs, k, d0, h=1e-4):
    n = X.size
    H = np.empty((n, n))
    for i in range(n):
        e = np.zeros(n)
        e[i] = h
        H[:, i] = -(_springs(X + e, pairs, k, d0)[1] - _springs(X - e, pairs, k, d0)[1]) / (2 * h)
    return H


def _spring_hessian(X, pairs, k):
    """Exact Hessian of springs at rest length (F = 0): k u u^T blocks."""
    X = X.reshape(-1, 3)
    H = np.zeros((X.size, X.size))
    for (a, b), kk in zip(pairs, k):
        u = X[a] - X[b]
        u = u / np.linalg.norm(u)
        K = kk * np.outer(u, u)
        for i, j, s in ((a, a, 1), (b, b, 1), (a, b, -1), (b, a, -1)):
            H[3 * i:3 * i + 3, 3 * j:3 * j + 3] += s * K
    return H


def test_diatomic_spring():
    m = np.array([1.00782503, 15.99491462])
    X = np.array([[0.1, -0.2, 0.3], [0.5, 0.4, 1.2]])
    k = 37.0  # eV / Angstrom^2
    r = vo.analyse(_spring_hessian(X, [(0, 1)], [k]), X, m)
    mu = m[0] * m[1] / m.sum()
    assert r['n_rigid'] == 5 and r['eig'].shape == (1,)
    assert abs(r['eig'][0] / (k / mu) - 1.0) < 1e-12
    hw = vo.HBAR * math.sqrt(k * vo.E_CHARGE * 1e20 / (mu * vo.AMU)) / vo.E_CHARGE  # hbar sqrt(k / mu) in SI
    assert abs(r['energies'][0] / hw - 1.0) < 1e-12
    # ASE's get_mode: the mass-weighted unit vector times m^-1/2, so sum_i m_i |mode_i|^2 = 1
    assert abs((m[:, None] * r['modes'][0] ** 2).sum() - 1.0) < 1e-12


def test_spring_network_against_central_differences():
    m = np.array([12.0, 1.008, 15.999])
    X = np.array([[0.0, 0.0, 0.0], [1.09, 0.0, 0.0], [-0.4, 1.15, 0.1]])
    pairs = [(0, 1), (0, 2), (1, 2)]
    d0 = [np.linalg.norm(X[a] - X[b]) for a, b in pairs]
    k = [30.0, 45.0, 5.0]
    H = _fd_hessian(X.ravel(), pairs, k, d0)
    r = vo.analyse(H, X, m)
    ref = np.linalg.eigh(vo.mass_weighted(H, m))[0]
    assert r['n_rigid'] == 6
    # at rest length the rigid modes are exact zeros of Hm; the FD Hessian is good to ~h^2 |E'''| / |E''|
    np.testing.assert_allclose(r['eig'], ref[6:], rtol=1e-6)
    assert np.all(np.abs(ref[:6]) < 1e-6 * ref[-1])


@pytest.mark.parametrize('shape, periodic, want', [('bent', False, 6), ('linear', False, 5), ('bent', True, 3),
                                                    ('atom', False, 3)])
def test_rigid_counts(shape, periodic, want):
    X = {'bent': np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [-0.3, 0.95, 0.0]]),
         'linear': np.array([[0.0, 0.0, 0.0], [1.1, 0.2, -0.3], [2.2, 0.4, -0.6]]),
         'atom': np.array([[0.3, 0.2, 0.1]])}[shape]
    m = np.linspace(1.0, 16.0, len(X))
    B = vo.rigid_basis(X, m, periodic)
    assert B.shape[0] == want
    np.testing.assert_allclose(B @ B.T, np.eye(want), atol=1e-14)
    Hp, k = vo.project(np.zeros((X.size, X.size)), X, m, periodic)
    assert k == want
    assert np.allclose(np.linalg.eigvalsh(Hp)[-want:], 1.0)  # c = 1 for a zero Hessian


def test_invariant_under_rigid_motion():
    rng = np.random.default_rng(3)
    m = np.array([12.0, 1.008, 1.008, 15.999])
    X = rng.standard_normal((4, 3))
    pairs = [(a, b) for a in range(4) for b in range(a)]
    k = rng.uniform(5.0, 40.0, len(pairs))
    f0 = vo.analyse(_spring_hessian(X, pairs, k), X, m)['frequencies']
    Q = np.linalg.qr(rng.standard_normal((3, 3)))[0]
    Y = X @ Q.T + rng.standard_normal(3)
    f1 = vo.analyse(_spring_hessian(Y, pairs, k), Y, m)['frequencies']
    np.testing.assert_allclose(f1, f0, rtol=1e-11)


def test_thermo_limits():
    from sgdml_b200 import vib

    e = np.array([0.01, 0.1, 0.4])
    zpe, U, S, F = vo.thermo(e, 1e-3)
    assert zpe == 0.5 * e.sum() and abs(U - zpe) < 1e-15 and abs(F - zpe) < 1e-15
    T = 1e7  # e / kT <= 5e-4: F per mode -> kT ln(e / kT) (the next term is kT (e / kT)^2 / 24)
    _, _, _, F = vo.thermo(e, T)
    kT = vo.KB_EV * T
    assert abs(F / (kT * np.log(e / kT)).sum() - 1.0) < 1e-7
    # the package's thermo on a result dict: imaginary and rigid slots excluded
    res = {'energies': np.array([[-0.02, 0.01, 0.1, 0.4, np.nan, np.nan]]), 'n_imaginary': np.array([1])}
    for T in (0.0, 1e-3, 300.0, 1e7):
        want = vo.thermo(e, T)
        got = vib.thermo(res, T)
        for k, w in zip(('zpe', 'U_vib', 'S_vib', 'F_vib'), want):
            # U - T S cancels at high T; the two evaluate exp(e / kT) - 1 differently (expm1 in the package)
            assert abs(got[k][0] - w) <= 1e-9 * max(abs(w), 1e-3), (T, k)
        assert got['n_excluded'][0] == 1


def test_vineyard_on_a_separable_quadratic_saddle():
    """Two atoms in a periodic cell (3 translations): the relative coordinate sees K = diag(k) at the minimum and
    diag(-k1', k2', k3') at the saddle, so nu_i = sqrt(k_i / mu) / 2 pi and the rate is closed form."""
    from sgdml_b200 import vib

    m = np.array([4.0, 12.0])
    mu = m.prod() / m.sum()
    X = np.array([[0.0, 0.0, 0.0], [1.5, 0.0, 0.0]])

    def H_of(K):
        return np.block([[np.diag(K), -np.diag(K)], [-np.diag(K), np.diag(K)]])

    kmin, ksad = np.array([10.0, 20.0, 30.0]), np.array([-7.0, 25.0, 35.0])
    a, b = vo.analyse(H_of(kmin), X, m, True), vo.analyse(H_of(ksad), X, m, True)
    assert a['n_rigid'] == 3 and b['n_rigid'] == 3 and (b['eig'] < 0).sum() == 1
    T, dE = 500.0, 0.3
    rate, pref = vo.vineyard(a['energies'], b['energies'], -1.0, -1.0 + dE, T)
    # nu = hbar omega / h (CODATA 2014 rounds hbar and h separately: h / 2 pi differs from hbar by 1e-10)
    nu = lambda k: vo.HBAR * math.sqrt(k * vo.E_CHARGE * 1e20 / (mu * vo.AMU)) / vo.HPLANCK  # noqa: E731
    pref_exact = nu(10.0) * nu(20.0) * nu(30.0) / (nu(25.0) * nu(35.0))
    assert abs(pref / pref_exact - 1.0) < 1e-12
    assert abs(rate / (pref_exact * math.exp(-dE / (vo.KB_EV * T))) - 1.0) < 1e-12

    def res(r, E):
        e = np.concatenate([r['energies'], [np.nan] * 3])[None]
        return {'energies': e, 'n_imaginary': np.array([(r['eig'] < 0).sum()]), 'n_rigid': np.array([3]),
                'potential_energy': np.array([E])}

    out = vib.harmonic_rate(res(a, -1.0), res(b, -1.0 + dE), T)
    assert abs(out['prefactor'][0] / pref_exact - 1.0) < 1e-12 and abs(out['rate'][0] / rate - 1.0) < 1e-12
    assert abs(out['barrier'][0] - dE) < 1e-15
    with pytest.raises(ValueError):
        vib.harmonic_rate(res(b, 0.0), res(b, dE), T)  # the minimum has an imaginary mode
    with pytest.raises(ValueError):
        vib.harmonic_rate(res(a, 0.0), res(a, dE), T)  # the saddle has none
    bad = res(b, dE)
    bad['n_rigid'] = np.array([5])
    with pytest.raises(ValueError):
        vib.harmonic_rate(res(a, 0.0), bad, T)
