"""The virial checks of tests/virial_checks.py on CPU: the oracle virial against an independent strain derivative of the
oracle energy, the free-molecule identity W = sum_i r_i F_i^T (and its failure once pairs wrap), and the componentwise
bound check_W, which an independent FP64 evaluation passes and each injected defect fails.  No GPU needed."""

import numpy as np
import pytest

import predict_checks as pc
import virial_checks as vc
from oracle import desc as odesc
from oracle import predict as opredict

N, M = 9, 23


def _cases():
    lat = pc.skewed_cell(N)
    return {
        'free': (vc.make_model(N, M, seed=3), None),
        'ecstr': (vc.make_model(N, M, seed=4, ecstr=True), None),
        'pbc': (vc.make_model(N, M, seed=5, lattice=lat), lat),
    }


@pytest.fixture(scope='module')
def cases():
    out = {}
    for name, (model, lat) in _cases().items():
        op = opredict.Predictor(model)
        R = vc.queries(N, 6, 40 + len(out), lat)
        out[name] = (model, op, R)
    return out


def _wraps(R, lat):
    _, c = pc._pair_frac(R, np.linalg.inv(lat))
    return np.mean(np.any(np.around(c) != 0, axis=-1))


@pytest.mark.parametrize('name', ['free', 'ecstr', 'pbc'])
def test_oracle_fdesc_gives_the_oracle_forces(cases, name):
    """The restated F_desc is the oracle's: std J^T F_desc equals oracle.predict's F."""
    model, op, R = cases[name]
    E, F, W, Fd = vc.oracle_virial(op, R)
    _, g = odesc.from_R(R, op.lat_and_inv)
    F2 = op.std * odesc.vec_dot_d_desc(g, Fd)
    assert np.max(np.abs(F2 - F)) <= 1e-13 * np.max(np.abs(F))


# measured max |W - W_strain| / max |W| at h = 1e-4 with Richardson extrapolation: 5.2e-12 (free), 1.6e-9 (ecstr),
# 1.2e-11 (pbc, skewed cell, >= 20 % of the pairs wrapped)
STRAIN_TOL = 1e-8


@pytest.mark.parametrize('name', ['free', 'ecstr', 'pbc'])
def test_oracle_virial_is_the_strain_derivative(cases, name):
    """W against central differences of the oracle energy under the six strains, the cell strained with the positions.
    The periodic case really wraps, so the image term L rint(L^-1 d) is part of what is checked."""
    model, op, R = cases[name]
    if name == 'pbc':
        assert _wraps(R, op.lat_and_inv[0]) >= 0.2
    W = vc.oracle_virial(op, R)[2]
    Ws = vc.strain_virial(op, R)
    rel = np.max(np.abs(W - Ws)) / np.max(np.abs(W))
    print('\n[virial] %s: oracle W vs strain derivative of E: max|dW|/max|W| %.1e' % (name, rel))
    assert rel < STRAIN_TOL
    assert np.max(np.abs(W - np.transpose(W, (0, 2, 1)))) <= 1e-12 * np.max(np.abs(W))


@pytest.mark.parametrize('name', ['free', 'ecstr'])
def test_free_molecule_virial_is_classical(cases, name):
    model, op, R = cases[name]
    _, F, W, _ = vc.oracle_virial(op, R)
    Wc = vc.classical_virial(R, F)
    assert np.max(np.abs(W - Wc)) <= 1e-12 * np.max(np.abs(W))


def test_periodic_virial_is_not_classical(cases):
    """Once pairs wrap, sum_i r_i F_i^T misses the image term: the two differ by far more than rounding."""
    model, op, R = cases['pbc']
    _, F, W, _ = vc.oracle_virial(op, R)
    Wc = vc.classical_virial(R, F)
    assert np.max(np.abs(W - Wc)) >= 1e-2 * np.max(np.abs(W))


def _k(model, op):
    return pc.n_terms(model['R_desc'].shape[1], op.n_perms, model['R_desc'].shape[0])


@pytest.mark.parametrize('name', ['free', 'ecstr', 'pbc'])
def test_check_W_passes_independent_evaluation(cases, name):
    """A second FP64 evaluation of the same sum, with the pair factor delta delta^T / |delta|^3 taken from the pair
    vectors instead of g_d delta_d^T, passes with a 10x margin."""
    model, op, R = cases[name]
    _, _, W, Fd = vc.oracle_virial(op, R)
    delta = vc.pair_vectors(R, op.lat_and_inv)
    dist = np.sqrt(np.sum(delta * delta, axis=-1))
    W2 = -op.std * np.einsum('bd,bdi,bdj->bij', Fd / dist ** 3, delta, delta)
    k = _k(model, op)
    r = vc.check_W(W2, W, vc.virial_abs_scale(model, R, op), k, what=name)
    print('\n[virial bound] %s independent: max|err|/scale %.2e, tau %.2e' % (name, r, pc.tau(k)))
    assert r <= pc.tau(k) / 10


def _defect(name, model, op, R):
    """W of the oracle with one defect injected."""
    lat_and_inv = op.lat_and_inv
    x, g = odesc.from_R(R, lat_and_inv)
    delta = vc.pair_vectors(R, lat_and_inv)
    Fd = np.array([vc.oracle_fdesc(op, xi) for xi in x])
    if name == 'unwrapped_delta':
        return vc.virial_from(Fd, g, vc.pair_vectors(R, None), op.std)
    if name == 'std_missing':
        return vc.virial_from(Fd, g, delta, 1.0)
    if name == 'split_plane_dropped':
        # the training points of one main-kernel split (here: one tile of 8 points) missing from F_desc
        q = vc.with_cell(op, None if lat_and_inv is None else lat_and_inv[0])
        S = op.n_perms
        keep = np.ones(op.R_desc_perms.shape[0], dtype=bool)
        keep[8 * S:16 * S] = False
        q.R_desc_perms = op.R_desc_perms[keep]
        q.R_d_desc_alpha_perms = op.R_d_desc_alpha_perms[keep]
        if op.alphas_E_lin is not None:
            q.alphas_E_lin = op.alphas_E_lin[keep]
        Fd2 = np.array([vc.oracle_fdesc(q, xi) for xi in x])
        return vc.virial_from(Fd2, g, delta, op.std)
    if name == 'pair_dropped':
        t = np.abs(Fd) * np.sum(np.abs(g), axis=-1) * np.sqrt(np.sum(delta * delta, axis=-1))
        Fd2 = Fd.copy()
        Fd2[:, int(np.argmax(np.max(t, axis=0)))] = 0.0
        return vc.virial_from(Fd2, g, delta, op.std)
    if name == 'transposed_sign_flipped':
        W = np.transpose(vc.virial_from(Fd, g, delta, op.std), (0, 2, 1)).copy()
        W[:, 0, 1] = -W[:, 0, 1]
        return W
    if name == 'cell_as_rows':
        lat = lat_and_inv[0].T
        li = (lat, np.linalg.inv(lat))
        q = vc.with_cell(op, lat)
        x2, g2 = odesc.from_R(R, li)
        Fd2 = np.array([vc.oracle_fdesc(q, xi) for xi in x2])
        return vc.virial_from(Fd2, g2, vc.pair_vectors(R, li), op.std)
    raise ValueError(name)


DEFECTS = ['unwrapped_delta', 'std_missing', 'split_plane_dropped', 'pair_dropped', 'transposed_sign_flipped',
           'cell_as_rows']


@pytest.mark.parametrize('defect', DEFECTS)
def test_check_W_fails_defects(cases, defect):
    name = 'pbc' if defect in ('unwrapped_delta', 'cell_as_rows') else 'ecstr'
    model, op, R = cases[name]
    W = vc.oracle_virial(op, R)[2]
    Wbad = _defect(defect, model, op, R)
    with pytest.raises(AssertionError):
        vc.check_W(Wbad, W, vc.virial_abs_scale(model, R, op), _k(model, op), what=defect)
