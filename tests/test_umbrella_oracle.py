"""The NumPy restatement of umbrella sampling (tests/umbrella_oracle.py) on CPU: the restraint's gradient and bias
force, the reduction to plain MD, continuation, the velocity correction of an exchange, and MBAR against the closed
forms of a harmonic oscillator."""

import numpy as np

import md_oracle
import umbrella_oracle as uo
from md_common import _spring_pes

CVS = [('distance', (0, 1)), ('angle', (1, 2, 3)), ('dihedral', (0, 2, 3, 4)), ('dihedral', (4, 3, 1, 0))]


def _geometries(n, seed=0):
    from sgdml_b200 import synth

    rng = np.random.default_rng(seed)
    return synth.base_geometry(5).reshape(1, 15) + 0.1 * rng.standard_normal((n, 15))


def _restraint_energy(R, cvs, c, kappa):
    X = R.reshape(-1, 5, 3)
    import metad_oracle

    s = np.stack([metad_oracle.cv_eval(k, a, X)[0] for k, a in cvs], 1)
    return uo.restraint(s, [k for k, _ in cvs], c, kappa)[0]


def test_restraint_gradient_matches_central_differences():
    R = _geometries(3)
    import metad_oracle

    s0 = np.stack([metad_oracle.cv_eval(k, a, R.reshape(-1, 5, 3))[0] for k, a in CVS], 1)
    kappa = np.array([3.0, 2.0, 1.5, 0.7])
    # the dihedral centres sit just inside +-pi on the far side of the current angles: the wrap is in play
    for c in (s0[0] + np.array([0.1, -0.2, 0.3, -0.1]), np.array([1.0, 1.5, np.pi - 1e-3, -np.pi + 1e-3])):
        _, b, Fb, _ = uo.bias(R, CVS, c[None], kappa[None], np.zeros(len(R), dtype=int))
        assert np.allclose(b, _restraint_energy(R, CVS, c, kappa), rtol=0, atol=0)
        eps = 1e-6
        for i in range(R.shape[1]):
            d = np.zeros(R.shape[1])
            d[i] = eps
            num = (_restraint_energy(R + d, CVS, c, kappa) - _restraint_energy(R - d, CVS, c, kappa)) / (2 * eps)
            assert np.allclose(-Fb[:, i], num, rtol=1e-6, atol=1e-7), i


def test_dihedral_difference_wraps():
    b, u = uo.restraint(np.array([[np.pi - 0.1]]), ['dihedral'], np.array([-np.pi + 0.1]), np.array([2.0]))
    assert np.isclose(u[0, 0], 2.0 * -0.2) and np.isclose(b[0], 0.5 * 2.0 * 0.04)


def test_bias_force_has_no_net_force_or_torque():
    R = _geometries(4, seed=1)
    C, K = np.array([[1.0, 2.0, 0.5, -2.5]]), np.array([[4.0, 3.0, 2.0, 1.0]])
    _, _, Fb, _ = uo.bias(R, CVS, C, K, np.zeros(4, dtype=int))
    F = Fb.reshape(-1, 5, 3)
    X = R.reshape(-1, 5, 3)
    assert np.max(np.abs(F.sum(1))) < 1e-12
    assert np.max(np.abs(np.cross(X, F).sum(1))) < 1e-11


def _spring_forces(R):
    E, F = _spring_pes(R)
    return E, F.reshape(R.shape)


def _state(n_rep, seed=3):
    R = _geometries(n_rep, seed)
    V = 0.01 * np.random.default_rng(seed + 1).standard_normal(R.shape)
    s = np.full(15, 0.5)
    return R, V, s


def test_zero_force_constants_without_exchange_are_md():
    R, V, s = _state(6)
    C, K = np.array([[1.0, 2.0], [1.2, 1.8], [1.4, 1.6]]), np.zeros((3, 2))
    fin, fr, _ = uo.run(_spring_forces, R, V, s, CVS[:2], C, K, 12, 0.05, 0.3, 0.02, 0, seed=5, step0=7, stride=3)
    (R1, V1, F1, E1), ref = md_oracle.run(_spring_forces, R, V, s, 12, 0.05, 0.3, 0.02, seed=5, step0=7, stride=3)
    for k in ref:
        assert np.array_equal(fr[k], ref[k]), k
    assert np.array_equal(fin['R'], R1) and np.array_equal(fin['V'], V1) and np.array_equal(fin['F'], F1)
    assert np.all(fr['bias'] == 0.0)


def test_two_runs_are_one_long_run():
    R, V, s = _state(8)
    C = np.array([[1.0, 1.9], [1.1, 1.8], [1.2, 1.7], [1.3, 1.6]])
    K = np.full((4, 2), 40.0)
    args = (s, CVS[:2], C, K)
    kw = dict(dt=0.05, gamma=0.3, kT=0.05, every=2, seed=11)
    a, fa, sa = uo.run(_spring_forces, R, V, *args, 20, step0=4, stride=2, **kw)
    b1, f1, s1 = uo.run(_spring_forces, R, V, *args, 10, step0=4, stride=2, **kw)
    b2, f2, s2 = uo.run(_spring_forces, b1['R'], b1['V'], *args, 10, step0=14, stride=2, walker=b1['walker'], **kw)
    for k in fa:
        assert np.array_equal(fa[k], np.concatenate([f1[k], f2[k]])), k
    assert np.array_equal(sa['n_attempted'], s1['n_attempted'] + s2['n_attempted'])
    assert np.array_equal(sa['n_accepted'], s1['n_accepted'] + s2['n_accepted'])
    assert sa['n_accepted'].sum() > 0  # exchanges are in play
    for w in fa['walker']:
        assert sorted(w[:4]) == [0, 1, 2, 3] and sorted(w[4:]) == [4, 5, 6, 7]


def test_exchange_keeps_each_configurations_full_step_velocity():
    R, V, s = _state(4)
    C, K = np.array([[1.0], [1.05], [1.1], [1.15]]), np.full((4, 1), 5.0)
    st = {'R': R.copy(), 'V': V.copy(), 'walker': np.arange(4, dtype=np.int32)}
    uo.evaluate(st, _spring_forces, CVS[:1], C, K)
    before = {k: np.array(v) for k, v in st.items()}
    stats = {'n_accepted': np.zeros((1, 3), dtype=np.int64), 'n_attempted': np.zeros((1, 3), dtype=np.int64),
             'margin': np.inf}
    uo.exchange(st, 2, 1, 0, 1.0 / 1e3, 0.025, s, CVS[:1], C, K, stats)  # hot: every swap is accepted
    assert np.array_equal(stats['n_accepted'], [[1, 0, 1]])
    for a, b in ((0, 1), (2, 3)):
        for x, y in ((a, b), (b, a)):
            assert np.array_equal(st['R'][x], before['R'][y]) and st['walker'][x] == before['walker'][y]
            # w - k + k with k = h (F_new s): within the rounding of the larger of w and k
            kn = 0.025 * (st['F'][x] * s)
            bound = np.spacing(np.maximum(np.abs(kn), np.abs(before['V'][y])))
            assert np.all(np.abs(st['V'][x] - before['V'][y]) <= 2 * bound)
            assert not np.array_equal(st['F'][x], before['F'][y])  # the new window's force
    # the device form: v = w - h (F_old s) moved, v' = w - h (F_new s)
    h = 0.025
    w = before['V'][1]
    v_dev = w - h * (st['F'][0] * s)
    assert np.array_equal(st['V'][0], v_dev + h * (st['F'][0] * s))


# ------------------------------------------------------------------------------------------------------------- MBAR
def _oscillator(k0, kappa, c, beta, n, rng):
    """samples of x under U = k0 x^2 / 2 + kappa (x - c)^2 / 2 (exact: a Gaussian), and the closed-form reduced free
    energy -ln Z up to a constant common to every window"""
    prec = beta * (k0 + kappa)
    mean = kappa * c / (k0 + kappa)
    x = mean + rng.standard_normal(n) / np.sqrt(prec)
    f = 0.5 * np.log(prec / (2 * np.pi)) + beta * k0 * kappa * c * c / (2 * (k0 + kappa))
    return x, f


def test_mbar_matches_the_harmonic_oscillator():
    """Eight windows along a harmonic well, 20 000 exact samples each: the window free energies within 0.05 kT of the
    closed form and the unbiased PMF within 0.1 kT of k0 x^2 / 2.  Neighbouring windows lie 1.4 standard deviations
    apart; over seeds 0 to 2 the largest deviation of f was 0.016 to 0.027 kT (the error accumulates along the
    windows), so the bound is about twice the statistical error."""
    rng = np.random.default_rng(0)
    k0, kappa, beta, n = 1.0, 10.0, 1.0, 20000
    centres = np.linspace(-1.5, 1.5, 8)
    xs, fs = zip(*(_oscillator(k0, kappa, c, beta, n, rng) for c in centres))
    x = np.concatenate(xs)
    u = np.array([beta * uo.restraint(x[:, None], ['distance'], [c], [kappa])[0] for c in centres])
    f, log_w, it = uo.mbar(u, [n] * 8, tol=1e-8)
    ref = np.array(fs) - fs[0]
    assert np.max(np.abs(f - ref)) < 0.05, (f, ref)
    assert abs(np.exp(log_w).sum() - 1.0) < 1e-12
    edges = np.linspace(-1.5, 1.5, 16)
    p, _ = np.histogram(x, edges, weights=np.exp(log_w))
    mid = 0.5 * (edges[1:] + edges[:-1])
    pmf = -np.log(p) / beta
    exact = 0.5 * k0 * mid**2
    d = (pmf - pmf.min()) - (exact - exact.min())
    assert np.max(np.abs(d - d.mean())) < 0.1, d
    # the unbiased mean of x^2 against 1 / (beta k0)
    assert abs(np.sum(np.exp(log_w) * x * x) - 1.0 / (beta * k0)) < 0.05


def test_mbar_one_window_is_zero():
    x = np.random.default_rng(1).standard_normal(1000)
    u = np.array([uo.restraint(x[:, None], ['distance'], [0.3], [2.0])[0]])
    f, log_w, it = uo.mbar(u, [1000])
    assert f.shape == (1,) and f[0] == 0.0 and it == 1
    w = np.exp(log_w)
    assert abs(w.sum() - 1.0) < 1e-12 and np.allclose(w, np.exp(u[0]) / np.exp(u[0]).sum(), rtol=1e-10)
