"""CPU: the NumPy restatement of the posterior covariance (tests/posterior_oracle.py) on every golden fixture with
training data.  It pins the conventions the device path follows: the mean of the same Gaussian process is the model's
prediction, the posterior at a training point is bounded by the noise lam, adding data never adds variance, the
Cholesky route agrees with a dense solve, and a^2 is the maximum-likelihood amplitude."""

import numpy as np
import pytest
import scipy.optimize

from conftest import load_golden

import oracle.predict as opredict
import oracle.train as otrain
import posterior_oracle as po

TOL = 1e-4  # eigenvalue bounds, in units of lam: the rounding of P - V V^T is ~1e-7 lam on these fixtures


def _case(name):
    g = load_golden(name)
    task = po.fixture_task(g)
    model = otrain.train(task)
    M = task['R_train'].shape[0]
    Rq = np.vstack((g['R_query'], task['R_train'].reshape(M, -1)))
    return g, task, model, Rq


@pytest.mark.parametrize('name', po.POSTERIOR_FIXTURES)
def test_mean_identity(name):
    """-std C(F_q, X) alpha is the predictor's F and +std C(E_q, X) alpha its E - c, to 1e-12 of the magnitude of
    the terms summed (alpha is large where C_XX + lam I is ill-conditioned, so the sum cancels)."""
    g, task, model, Rq = _case(name)
    J = po.Joint(task, Rq, 'alphas_E' in model)
    alpha = np.asarray(model['alphas_F'], dtype=np.float64).ravel()
    if 'alphas_E' in model:
        alpha = np.hstack((alpha, model['alphas_E']))
    std = float(model['std'])
    E, F = opredict.Predictor(model).predict(Rq)
    for q, qi in enumerate(J.queries):
        CF, CE = J.C[np.ix_(qi[:-1], J.train)], J.C[qi[-1], J.train]
        assert np.all(np.abs(-std * CF @ alpha - F[q]) <= 1e-12 * std * (np.abs(CF) @ np.abs(alpha)))
        assert abs(std * CE @ alpha - (E[q] - model['c'])) <= 1e-12 * std * (np.abs(CE) @ np.abs(alpha))


@pytest.mark.parametrize('name', po.POSTERIOR_FIXTURES)
def test_training_point_bound_and_monotonicity(name):
    """At a training geometry the observed outputs' normalised posterior is lam C (C + lam I)^-1: eigenvalues in
    [0, lam] (the force block, or the whole block with energy constraints).  Dropping a training point never lowers
    any query's normalised posterior in the Loewner order."""
    g, task, model, Rq = _case(name)
    lam = float(model['lam'])
    J = po.Joint(task, Rq, 'alphas_E' in model)
    S = po.normalised_blocks(J, lam)
    B0, M = g['R_query'].shape[0], task['R_train'].shape[0]
    for m in range(M):
        blk = S[B0 + m] if 'alphas_E' in model else S[B0 + m][:-1, :-1]
        ev = np.linalg.eigvalsh(blk)
        assert ev.min() >= -TOL * lam and ev.max() <= lam * (1 + TOL), (m, ev.min(), ev.max())
    S_drop = po.normalised_blocks(J, lam, train=J.without(M // 2))
    for q in range(len(J.queries)):
        assert np.linalg.eigvalsh(S_drop[q] - S[q]).min() >= -TOL * lam


@pytest.mark.parametrize('name', po.POSTERIOR_FIXTURES)
def test_cholesky_route_matches_dense_solve(name):
    g, task, model, Rq = _case(name)
    J = po.Joint(task, Rq, 'alphas_E' in model)
    lam = float(model['lam'])
    S = po.normalised_blocks(J, lam)
    S_dense = po.normalised_blocks(J, lam, route='dense')
    P = np.array([J.C[np.ix_(qi, qi)] for qi in J.queries])
    A = J.C[np.ix_(J.train, J.train)] + lam * np.eye(len(J.train))
    bound = 8 * len(J.train) * np.finfo(float).eps * np.linalg.cond(A) ** 0.5 * np.abs(np.diagonal(P, axis1=1, axis2=2)).max()
    assert np.max(np.abs(S - S_dense)) <= bound


def test_amplitude_maximises_likelihood():
    """a^2 = |L^-1 y|^2 / n maximises the Gaussian log-likelihood of y under the covariance a^2 (C_XX + lam I)."""
    g, task, model, Rq = _case('n9_m16_s6')
    J = po.Joint(task, Rq[:1], False)
    a2 = po.amplitude(J, task, float(model['lam']))
    y = otrain.labels(task)[0]
    A = J.C[np.ix_(J.train, J.train)] + float(model['lam']) * np.eye(len(J.train))
    quad = float(y @ np.linalg.solve(A, y))

    def nll(log_a2):  # -log p(y | a^2) up to a constant
        return 0.5 * (quad / np.exp(log_a2) + len(y) * log_a2)

    res = scipy.optimize.minimize_scalar(nll, bracket=(np.log(a2) - 3, np.log(a2) + 3), tol=1e-12)
    assert abs(np.exp(res.x) / a2 - 1) < 1e-6
    # and Sigma is a^2 std^2 times the normalised blocks, E-F entries negated
    Sig, a2_p, _ = po.posterior(model, task, Rq[:2])
    S = po.normalised_blocks(po.Joint(task, Rq[:2], False), float(model['lam']))
    assert a2_p == a2
    assert np.allclose(Sig, a2 * float(model['std']) ** 2 * po.flip_energy(S), rtol=0, atol=0)


def test_labels_helper_matches_training():
    """GDMLTrain.train builds y with sgdml_b200.train.labels; the oracle's restatement gives the same vector."""
    from sgdml_b200.train import labels

    for name in ('n9_m16_s6', 'ecstr_n6_m8'):
        task = po.fixture_task(load_golden(name))
        y, std, mean = labels(task, bool(task['use_E_cstr']))
        y_o, std_o, mean_o = otrain.labels(task)
        assert np.array_equal(y, y_o) and std == std_o and mean == mean_o
