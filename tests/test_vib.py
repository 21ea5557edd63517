"""Normal modes on the device: sgdml_b200_vib_project against tests/vib_oracle.py, the batched Jacobi eigensolver against
numpy.linalg.eigh on planted spectra, and GDMLVibrations end to end: the minima and the CI-NEB saddle of the double-well
hinge model of test_neb.py, a golden model against a central-difference Hessian of its forces, a periodic model and a
geometry above the eigensolver's cap."""

import numpy as np
import pytest

import hvp_oracle
import vib_oracle as vo

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


def _cuda(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64)).cuda()


def _project(H, R, masses, periodic):
    import torch

    from sgdml_b200 import _lib

    B, n = H.shape[0], H.shape[1]
    Hd, Rd, ism = _cuda(H), _cuda(R), _cuda(np.asarray(masses) ** -0.5)
    Hp = torch.empty_like(Hd)
    k = torch.empty(B, dtype=torch.int64, device='cuda')
    _lib.check(_lib.lib().sgdml_b200_vib_project(_lib.ptr(Hd), _lib.ptr(Rd), _lib.ptr(ism), B, n // 3, periodic,
                                                 _lib.ptr(Hp), _lib.ptr(k), _lib.current_stream()), 'vib_project')
    return Hp.cpu().numpy(), k.cpu().numpy()


@pytest.mark.parametrize('shape, periodic', [('bent', 0), ('linear', 0), ('bent', 1)])
def test_projection_against_oracle(shape, periodic):
    rng = np.random.default_rng(4)
    N, B = 7, 3
    R = rng.standard_normal((B, N, 3))
    if shape == 'linear':
        R = rng.standard_normal((B, 1, 3)) * np.linspace(-2.0, 2.0, N)[None, :, None] + rng.standard_normal((B, 1, 3))
    m = rng.uniform(1.0, 20.0, N)
    H = rng.standard_normal((B, 3 * N, 3 * N))  # not symmetric: the projection symmetrises
    Hp, k = _project(H, R.reshape(B, -1), m, periodic)
    for b in range(B):
        want, kw = vo.project(H[b], R[b], m, bool(periodic))
        assert k[b] == kw == (3 if periodic else 5 if shape == 'linear' else 6)
        assert np.array_equal(Hp[b], Hp[b].T)
        assert np.max(np.abs(Hp[b] - want)) < 1e-12 * np.max(np.abs(want))


def _planted(n, seed):
    """A random symmetric n x n matrix with a planted spectrum of clusters (degenerate to the last bit), spread over 6
    orders of magnitude and both signs, and its eigenvalues."""
    rng = np.random.default_rng(seed)
    lam = rng.choice([-1.0, 1.0], n) * 10.0 ** rng.uniform(-3, 3, n)
    if n >= 4:
        lam[: n // 4] = lam[0]  # a degenerate cluster
        lam[n // 4: n // 4 + 2] = 0.0
    Q = np.linalg.qr(rng.standard_normal((n, n)))[0]
    A = (Q * lam) @ Q.T
    return 0.5 * (A + A.T), np.sort(lam)


@pytest.mark.parametrize('n', [1, 2, 31, 32, 33, 63, 126, 160])
def test_symeig_against_numpy(n):
    """Eigenvalues within 4 n eps |A|_2 of numpy's; |V^T V - I| and |A V - V diag(w)| / |A|_2 within 4 n eps
    (max-norm); two calls bit-identical."""
    from sgdml_b200 import _lib, vib

    assert _lib.lib().sgdml_b200_symeig_max_n() == 160
    B = 8
    mats = [_planted(n, 10 * n + b) for b in range(B)]
    A = np.stack([a for a, _ in mats])
    w, V = vib.symeig(_cuda(A))
    w, V = w.cpu().numpy(), V.cpu().numpy()
    w2, V2 = vib.symeig(_cuda(A))
    assert np.array_equal(w, w2.cpu().numpy()) and np.array_equal(V, V2.cpu().numpy())
    worst = [0.0, 0.0, 0.0]
    for b in range(B):
        a = A[b]
        ref = np.linalg.eigvalsh(a)
        nrm = max(np.max(np.abs(ref)), 1e-300)
        assert np.all(np.diff(w[b]) >= 0)
        e = [np.max(np.abs(w[b] - ref)) / nrm, np.max(np.abs(V[b].T @ V[b] - np.eye(n))),
             np.max(np.abs(a @ V[b] - V[b] * w[b])) / nrm]
        worst = [max(x, y) for x, y in zip(worst, e)]
    print('n %d: eigenvalue, orthogonality, residual errors in units of n eps: %s' % (n, np.array(worst) / (n * EPS)))
    assert max(worst) < 4 * n * EPS


def test_symeig_rejects_bad_calls():
    from sgdml_b200 import _lib

    import torch

    L = _lib.lib()
    A = _cuda(np.eye(4)[None])
    w = torch.full((1, 4), 7.0, dtype=torch.float64, device='cuda')
    V = torch.full((1, 4, 4), 7.0, dtype=torch.float64, device='cuda')
    s = _lib.current_stream()
    for n in (0, 161):
        assert L.sgdml_b200_symeig_batched(_lib.ptr(A), n, 1, _lib.ptr(w), _lib.ptr(V), s) <= -1000
    host = np.eye(4)
    assert L.sgdml_b200_symeig_batched(host.ctypes.data, 4, 1, _lib.ptr(w), _lib.ptr(V), s) <= -1000
    assert L.sgdml_b200_symeig_batched(_lib.ptr(A), 4, 1, _lib.ptr(w), _lib.ptr(A), s) <= -1000
    assert bool((w == 7.0).all()) and bool((V == 7.0).all())
    assert L.sgdml_b200_symeig_batched(_lib.ptr(A), 4, 0, _lib.ptr(w), _lib.ptr(V), s) == 0


def test_golden_model_against_central_differences():
    """Frequencies from predict_hessian against those of a central-difference Hessian of predict's forces.  The step
    h = 1e-4 Angstrom leaves a truncation error of h^2 |F'''| / 6 (~1e-8 relative to |H| on these smooth models) and a
    rounding error of eps |F| / h (~1e-12 relative), so 1e-6 relative on each eigenvalue of the mass-weighted Hessian
    (|H| sets the scale) is loose by two orders."""
    import sgdml_b200

    model, Rq, _ = hvp_oracle.fixture_model('n9_m16_s6')
    N = 9
    m = np.linspace(1.0, 16.0, N)
    vib = sgdml_b200.GDMLVibrations(model, m, E_to_eV=1.0, F_to_eV_Ang=1.0)
    X = Rq[:2].reshape(2, N, 3)
    res = vib.analyse(X)
    gp = vib.gdml_predict
    h = 1e-4
    for b in range(2):
        H = np.empty((3 * N, 3 * N))
        for i in range(3 * N):
            d = np.zeros(3 * N)
            d[i] = h
            _, Fp = gp.predict((X[b].ravel() + d)[None])
            _, Fm = gp.predict((X[b].ravel() - d)[None])
            H[:, i] = -(Fp[0] - Fm[0]) / (2 * h)
        ref = vo.analyse(H, X[b], m)
        k = int(res['n_rigid'][b])
        assert k == ref['n_rigid'] == 6
        w = np.sign(res['energies'][b, :-k]) * (res['energies'][b, :-k] / vo.EV_PER_SQRT_EIG) ** 2
        scale = np.max(np.abs(vo.mass_weighted(H, m)))
        assert np.max(np.abs(w - ref['eig'])) < 1e-6 * scale
        assert np.all(np.isnan(res['frequencies'][b, -k:])) and res['n_imaginary'][b] == (ref['eig'] < 0).sum()
        # the device result against the oracle on the same Hessian
        same = vo.analyse(res['hessian'][b], X[b], m)
        assert np.max(np.abs(w - same['eig'])) < 1e-9 * scale
        assert abs(res['zpe'][b] - 0.5 * same['energies'][same['energies'] > 0].sum()) < 1e-9 * res['zpe'][b]
        assert np.isclose(res['fmax'][b], np.max(np.linalg.norm(gp.predict(X[b].reshape(1, -1))[1].reshape(N, 3), axis=1)))


def test_periodic_and_above_the_cap():
    """A periodic model keeps 3 rigid modes; 60 atoms (n = 180 > 160) take torch.linalg.eigh on the same matrices."""
    import torch

    import sgdml_b200

    model, Rq, _ = hvp_oracle.fixture_model('pbc_n6_m8')
    vib = sgdml_b200.GDMLVibrations(model, np.full(6, 12.0))
    res = vib.analyse(_cuda(Rq[:3].reshape(3, 6, 3)))
    assert res['frequencies'].is_cuda and torch.all(res['n_rigid'] == 3)
    assert torch.all(torch.isfinite(res['frequencies'][:, :15])) and torch.all(torch.isnan(res['frequencies'][:, 15:]))
    model, Rq, _ = hvp_oracle.fixture_model('big_c60_m2_s120')
    vib = sgdml_b200.GDMLVibrations(model, np.full(60, 12.0))
    res = vib.analyse(Rq[:1].reshape(1, 60, 3))
    assert res['n_rigid'][0] == 6 and res['modes'].shape == (1, 180, 60, 3)
    same = vo.analyse(res['hessian'][0], Rq[0].reshape(60, 3), np.full(60, 12.0))
    w = np.sign(res['energies'][0, :-6]) * (res['energies'][0, :-6] / vo.EV_PER_SQRT_EIG) ** 2
    assert np.max(np.abs(w - same['eig'])) < 1e-9 * np.max(np.abs(same['eig']))


def test_minima_and_saddle_of_the_double_well_hinge():
    """The model of test_neb.py's double-well hinge: relaxed minima have no imaginary mode, the CI-NEB climbing image
    exactly one, whose mode lies along the band's tangent at the climbing image, and the Vineyard rate is finite."""
    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc
    from test_neb import _DW_PHI, _dw_hinge, _dw_task

    model = sgdml_b200.GDMLTrain().train(_dw_task())
    gp = sgdml_b200.GDMLPredict(model)
    dt, dtmax = 0.01 / np.sqrt(kc), 0.05 / np.sqrt(kc)
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=2)
    mins = rel.relax(_dw_hinge(_DW_PHI), fmax=1e-4 * kc, max_steps=3000, optimizer='fire', maxstep=0.05, dt=dt,
                     dtmax=dtmax)
    assert mins['converged'].all()
    neb = sgdml_b200.GDMLNEB(gp, 9)
    band = neb.interpolate(mins['positions'][0], mins['positions'][1], align=True)
    k = 50.0 * kc
    neb.neb(band, fmax=0.05 * kc, max_steps=2000, k=k, climb=False, maxstep=0.05, dt=dt, dtmax=dtmax)
    ci = neb.neb(fmax=1e-6 * kc, max_steps=5000, k=k, climb=True, maxstep=0.05, dt=dt, dtmax=dtmax)
    assert ci['converged'].all()
    top = int(ci['climbing_image'][0])
    P = ci['positions'][0]

    m = np.full(4, 12.0)
    vib = sgdml_b200.GDMLVibrations(gp, m)
    a = vib.analyse(mins['positions'])
    s = vib.analyse(P[top][None])
    print('minima: %s cm^-1\nsaddle: %s cm^-1' % (a['frequencies'], s['frequencies']))
    assert np.all(a['n_rigid'] == 6) and np.all(a['n_imaginary'] == 0)
    assert s['n_rigid'][0] == 6 and s['n_imaginary'][0] == 1 and s['frequencies'][0, 0] < 0
    # the imaginary mode against the band's tangent at the climbing image (central difference of its neighbours),
    # compared in mass-weighted coordinates where the modes are orthonormal
    sm = np.repeat(np.sqrt(m), 3)
    mode = s['modes'][0, 0].ravel() * sm
    tan = (P[top + 1] - P[top - 1]).ravel() * sm
    cos = abs(mode @ tan) / (np.linalg.norm(mode) * np.linalg.norm(tan))
    print('|cos(imaginary mode, tangent)| = %.5f' % cos)
    assert cos > 0.99
    for b in range(2):
        r = sgdml_b200.harmonic_rate({key: v[b:b + 1] for key, v in a.items()}, s, 300.0)
        print('rate from minimum %d: %.3e s^-1, prefactor %.3e s^-1, barrier %.4f eV' % (
            b, r['rate'][0], r['prefactor'][0], r['barrier'][0]))
        assert np.isfinite(r['rate'][0]) and r['rate'][0] > 0 and r['barrier'][0] > 0
    t = sgdml_b200.thermo(a, 300.0)
    assert np.all(np.isfinite(t['F_vib'])) and np.all(t['n_excluded'] == 0)
