"""GPU: GDMLPosterior against the NumPy restatement (tests/posterior_oracle.py) and against LAPACK, the device's own
cross rows against the predictor, the training-point bound, chunk invariance and the constructor's refusals.

Models are trained on the device from each fixture's training geometries and labels; the large-molecule fixtures carry
no labels, so a synthetic task of the same shape (synth.make_task) stands in for them.

Bound on the blocks: |Sigma_dev - Sigma_ref| <= 8 n eps kappa_2(C_XX + lam I)^(1/2) max diag(P) a^2 std^2."""

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse.linalg

from conftest import load_golden

import posterior_oracle as po

pytestmark = pytest.mark.gpu

EPS = np.finfo(np.float64).eps
BIG = {'big_n240_m2_s3': True, 'big_n100_m2_s12': False, 'big_c60_m2_s120': False}  # name -> use_E_cstr
TOL = 1e-4  # training-point eigenvalue bound, in units of lam, or the error bound where that is larger

_cache = {}


def _task(name):
    from sgdml_b200 import synth

    g = load_golden(name)
    if name in BIG:
        N, M = int(g['n_atoms']), g['R_train'].shape[0]
        task = synth.make_task(N, M, g['perms'], int(g['sig']), lam=float(g['lam']))
        task['use_E_cstr'] = BIG[name]
    else:
        task = po.fixture_task(g)
    return g, task


def _trained(name):
    """(g, task, model, R_query): the model trained on the device; queries R_query and the training geometries."""
    if name not in _cache:
        import sgdml_b200

        g, task = _task(name)
        gt = sgdml_b200.GDMLTrain()
        model = gt.train(task)
        gt.release_buffers()
        M = task['R_train'].shape[0]
        Rq = np.vstack((g['R_query'], np.asarray(task['R_train']).reshape(M, -1)))
        _cache[name] = (g, task, model, Rq)
    return _cache[name]


def _alphas(model):
    a = np.asarray(model['alphas_F'], dtype=np.float64).ravel()
    return np.hstack((a, model['alphas_E'])) if 'alphas_E' in model else a


# the oracle's dense-Jacobian assembly takes minutes at 240 atoms (D = 28 680): that shape is covered by the mean
# identity on the device's own cross rows and by chunk invariance
@pytest.mark.parametrize('name', po.POSTERIOR_FIXTURES + ['big_n100_m2_s12', 'big_c60_m2_s120'])
def test_device_against_oracle(name):
    import sgdml_b200

    g, task, model, Rq = _trained(name)
    post = sgdml_b200.GDMLPosterior(model, task)
    cov = post.predict_cov(Rq)
    ref, a2, J = po.posterior(model, task, Rq)
    lam = float(model['lam'])
    A = J.C[np.ix_(J.train, J.train)] + lam * np.eye(len(J.train))
    P = np.array([J.C[np.ix_(qi, qi)] for qi in J.queries])
    scale = a2 * float(model['std']) ** 2
    bound = 8 * post.n * EPS * np.linalg.cond(A) ** 0.5 * np.diagonal(P, axis1=1, axis2=2).max() * scale
    ratio = np.max(np.abs(cov - ref)) / bound
    print('%s: worst |Sigma_dev - Sigma_oracle| / bound = %.3g, a2 %.6g vs %.6g' % (name, ratio, post.amplitude, a2))
    assert ratio <= 1.0
    assert abs(post.amplitude / a2 - 1) <= max(1e-8, 8 * post.n * EPS * np.linalg.cond(A))
    assert np.array_equal(cov, np.swapaxes(cov, 1, 2))  # exactly symmetric
    B0, M = Rq.shape[0] - task['R_train'].shape[0], task['R_train'].shape[0]
    # training-point bound on the device's own blocks, within the device's error bound (normalised)
    tol = max(TOL * lam, post.dim * bound / scale)  # |eigenvalue shift| <= |error|_F <= d max|error|
    for m in range(M):
        S = cov[B0 + m] / post.scale
        ev = np.linalg.eigvalsh(S if 'alphas_E' in model else S[:-1, :-1])
        assert ev.min() >= -tol and ev.max() <= lam + tol, (m, ev.min(), ev.max())
    E_std, F_std = post.predict_std(Rq)
    assert np.array_equal(E_std, np.sqrt(np.maximum(cov[:, -1, -1], 0)))
    assert np.array_equal(F_std, np.sqrt(np.maximum(np.diagonal(cov, axis1=1, axis2=2)[:, :-1], 0)))
    post.release()


@pytest.mark.parametrize('name', po.POSTERIOR_FIXTURES + list(BIG))
def test_device_cross_rows_reproduce_the_prediction(name):
    """-std C(F_q, X) alpha from the device's assembled cross rows is GDMLPredict's F, +std C(E_q, X) alpha its E - c,
    to 1e-12 of the magnitude of the terms summed."""
    import sgdml_b200

    g, task, model, Rq = _trained(name)
    post = sgdml_b200.GDMLPosterior(model, task)
    V, _P = post._cross_rows(np.ascontiguousarray(Rq))
    V = V[:, :post.n].cpu().numpy()
    B, n3 = Rq.shape[0], 3 * post.n_atoms
    alpha, std = _alphas(model), float(model['std'])
    E, F = sgdml_b200.GDMLPredict(model).predict(Rq)
    CF = V[:B * n3].reshape(B, n3, -1)
    CE = V[B * n3:]
    assert np.all(np.abs(-std * CF @ alpha - F) <= 1e-12 * std * (np.abs(CF) @ np.abs(alpha)))
    assert np.all(np.abs(std * CE @ alpha - (E - model['c'])) <= 1e-12 * std * (np.abs(CE) @ np.abs(alpha)))
    post.release()


@pytest.mark.parametrize('name', ['n9_m16_s6', 'ecstr_n6_m8', 'pbc_n6_m8', 'big_n240_m2_s3'])
def test_chunk_invariance(name):
    """Caps of 1 and 3 queries per chunk and no cap give bit-identical blocks, and torch input the same as NumPy."""
    import torch

    import sgdml_b200

    g, task, model, Rq = _trained(name)
    post = sgdml_b200.GDMLPosterior(model, task)
    ref = post.predict_cov(Rq)
    for cap in (1, 3):
        post._max_chunk = cap
        assert np.array_equal(post.predict_cov(Rq), ref), cap
    post._max_chunk = None
    assert np.array_equal(post.predict_cov(torch.from_numpy(Rq).cuda()), ref)
    assert np.array_equal(post.predict_cov(Rq[3]), ref[3:4])
    post.release()


def test_size_against_lapack():
    """N = 21, M = 261 (n = 16 443, odd, 129 TRSM blocks): the device's solved cross rows and blocks against
    scipy.linalg.cho_factor + solve_triangular on the device-assembled K."""
    import sgdml_b200
    from sgdml_b200 import synth

    N, M = 21, 261
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, 20)
    gt = sgdml_b200.GDMLTrain()
    model = gt.train(task)
    Rq = synth.geometries(N, 5, 7).reshape(5, -1)
    post = sgdml_b200.GDMLPosterior(model, task)
    n, d = post.n, post.dim
    assert n == 16443
    V_dev, P = post._solved_rows(np.ascontiguousarray(Rq))
    V_dev, P = V_dev[:, :n].cpu().numpy(), P.cpu().numpy()
    cov = post.predict_cov(Rq)
    Vc, _ = post._cross_rows(np.ascontiguousarray(Rq))
    Vc = Vc[:, :n].cpu().numpy()
    X, G = post.desc.from_R(task['R_train'].reshape(M, -1))
    A, _ = gt._assemble_kernel_mat_device(X, G, post.tril_perms_lin, post.sig, scale=-1.0)
    A = A[:, :n].cpu().numpy()
    gt.release_buffers()
    A[np.diag_indices_from(A)] += post.lam
    lam_max = scipy.sparse.linalg.eigsh(A, k=1, which='LA', return_eigenvectors=False)[0]
    kappa = lam_max / post.lam  # >= kappa_2: C_XX is positive semi-definite, so lambda_min >= lam
    Lf = np.tril(scipy.linalg.cho_factor(A, lower=True, overwrite_a=True)[0])
    del A
    V_ref = scipy.linalg.solve_triangular(Lf, Vc.T, lower=True).T
    bound = 8 * n * EPS * kappa ** 0.5 * np.diagonal(P, axis1=1, axis2=2).max()
    print('size: worst V ratio %.3g' % (np.max(np.abs(V_dev - V_ref)) / bound))
    assert np.max(np.abs(V_dev - V_ref)) <= bound
    rows = [np.hstack((np.arange(q * (d - 1), (q + 1) * (d - 1)), [5 * (d - 1) + q])) for q in range(5)]
    S_ref = po.flip_energy(np.array([P[q] - V_ref[r] @ V_ref[r].T for q, r in enumerate(rows)])) * post.scale
    print('size: worst Sigma ratio %.3g' % (np.max(np.abs(cov - S_ref)) / (bound * post.scale)))
    assert np.max(np.abs(cov - S_ref)) <= bound * post.scale
    post.release()


def test_refusals_and_release():
    import torch

    import sgdml_b200

    g, task, model, Rq = _trained('n9_m16_s6')
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()

    bad = dict(model, solver_name='cg')
    with pytest.raises(ValueError, match='analytic'):
        sgdml_b200.GDMLPosterior(bad, task)
    assert torch.cuda.memory_allocated() == before

    with pytest.raises(ValueError, match=r'release_buffers\(\)'):
        sgdml_b200.GDMLPosterior(model, task, max_memory=1e-6)
    assert torch.cuda.memory_allocated() == before

    moved = dict(task, R_train=task['R_train'] * 1.01)
    with pytest.raises(ValueError, match='descriptors'):
        sgdml_b200.GDMLPosterior(model, moved)
    assert torch.cuda.memory_allocated() == before

    F = np.array(task['F_train'], copy=True)
    F[0, 0, 0] += 0.5
    with pytest.raises(ValueError, match='coefficients'):
        sgdml_b200.GDMLPosterior(model, dict(task, F_train=F))
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    with pytest.raises(ValueError, match='coefficients'):
        sgdml_b200.GDMLPosterior(dict(model, lam=model['lam'] * 100), task)
    assert torch.cuda.memory_allocated() == before

    post = sgdml_b200.GDMLPosterior(model, task)
    post.predict_cov(Rq)
    assert torch.cuda.memory_allocated() > before
    post.release()
    assert torch.cuda.memory_allocated() == before
    with pytest.raises(RuntimeError, match='released'):
        post.predict_cov(Rq)
