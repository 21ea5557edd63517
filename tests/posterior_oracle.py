"""NumPy restatement of GDMLPosterior (sgdml_b200/posterior.py), independent of the device path.

The joint covariance C = -K_ref over the point set [training; queries] comes from oracle.assemble.assemble_E_cstr
(layout [forces; energies], energy rows for -E), the posterior from a Schur complement through
scipy.linalg.cho_factor / solve_triangular, and the amplitude a^2 = |L^-1 y|^2 / n from the same factor.
"""

import numpy as np
import scipy.linalg

import oracle.assemble as oassemble
import oracle.desc as odesc
import oracle.train as otrain

POSTERIOR_FIXTURES = ['n5_m10_s1', 'n9_m16_s6', 'n12_m8_s12', 'n21_m6_s6', 'ecstr_n6_m8', 'pbc_n6_m8']


def fixture_task(g):
    """The task a golden fixture with training data was trained on: its geometries, labels, sig, lam and cell."""
    task = {
        'type': 't', 'code_version': 'golden', 'dataset_name': 'golden', 'dataset_theory': 'golden',
        'z': np.asarray(g['z']), 'R_train': np.asarray(g['R_train'], dtype=np.float64),
        'F_train': np.asarray(g['F_train'], dtype=np.float64), 'E_train': np.asarray(g['E_train'], dtype=np.float64),
        'idxs_train': np.arange(g['R_train'].shape[0]), 'md5_train': b'0' * 32,
        'idxs_valid': np.arange(0), 'md5_valid': b'0' * 32,
        'sig': int(g['sig']), 'lam': float(g['lam']), 'use_E': True,
        'use_E_cstr': bool(g['use_E_cstr']) if 'use_E_cstr' in g else False, 'use_sym': True,
        'perms': np.asarray(g['perms'], dtype=np.int64),
    }
    if 'lattice' in g:
        task['lattice'] = np.asarray(g['lattice'], dtype=np.float64)
    return task


def _lat_and_inv(task_or_model):
    if 'lattice' not in task_or_model:
        return None
    lat = np.asarray(task_or_model['lattice'], dtype=np.float64)
    return lat, np.linalg.inv(lat)


class Joint(object):
    """C = -K_ref over [training; queries] and the index sets of the training columns and the query outputs."""

    def __init__(self, task, R_query, use_E_cstr):
        M, N = task['R_train'].shape[:2]
        lat_and_inv = _lat_and_inv(task)
        R_all = np.vstack((np.asarray(task['R_train'], dtype=np.float64).reshape(M, -1),
                           np.asarray(R_query, dtype=np.float64).reshape(-1, 3 * N)))
        X, G = odesc.from_R(R_all, lat_and_inv)
        tlin = odesc.tril_perms_lin(task['perms'])
        self.C = -oassemble.assemble_E_cstr(X, G, tlin, task['sig'])
        self.M, self.N, self.B = M, N, R_all.shape[0] - M
        n3, nf = 3 * N, 3 * N * R_all.shape[0]
        self.train = np.arange(n3 * M)
        if use_E_cstr:
            self.train = np.hstack((self.train, nf + np.arange(M)))
        self.queries = [np.hstack((np.arange(n3 * (M + q), n3 * (M + q + 1)), [nf + M + q])) for q in range(self.B)]

    def without(self, m):
        """The training columns with training point m left out."""
        n3 = 3 * self.N
        nf = n3 * (self.M + self.B)
        keep = np.where(self.train < nf, self.train // n3 != m, self.train != nf + m)
        return self.train[keep]


def normalised_blocks(J, lam, train=None, route='cholesky'):
    """S_q = P_q - C(z_q, X) (C_XX + lam I)^-1 C(X, z_q) for every query, in the assembled order [F; -E]."""
    tx = J.train if train is None else train
    A = J.C[np.ix_(tx, tx)] + lam * np.eye(len(tx))
    out = []
    if route == 'cholesky':
        Lf = scipy.linalg.cho_factor(A, lower=True)[0]
        Lf = np.tril(Lf)
        for qi in J.queries:
            W = scipy.linalg.solve_triangular(Lf, J.C[np.ix_(tx, qi)], lower=True)
            out.append(J.C[np.ix_(qi, qi)] - W.T @ W)
    else:
        for qi in J.queries:
            Cx = J.C[np.ix_(qi, tx)]
            out.append(J.C[np.ix_(qi, qi)] - Cx @ np.linalg.solve(A, Cx.T))
    return np.array(out)


def flip_energy(S):
    """[F; -E] -> [F; E]: negates the E-F entries."""
    S = np.array(S, copy=True)
    S[..., -1, :-1] *= -1
    S[..., :-1, -1] *= -1
    return S


def amplitude(J, task, lam):
    """a^2 = |L^-1 y|^2 / n with y the normalised labels train() solves for."""
    y, _std, _mean = otrain.labels(task)
    A = J.C[np.ix_(J.train, J.train)] + lam * np.eye(len(J.train))
    Lf = np.tril(scipy.linalg.cho_factor(A, lower=True)[0])
    z = scipy.linalg.solve_triangular(Lf, y, lower=True)
    return float(z @ z) / len(y)


def posterior(model, task, R_query):
    """(Sigma (B, d, d) in [F; E] order and the model's units squared, a^2, the Joint)."""
    use_E_cstr = 'alphas_E' in model
    J = Joint(task, R_query, use_E_cstr)
    lam = float(model['lam'])
    a2 = amplitude(J, task, lam)
    S = normalised_blocks(J, lam)
    return a2 * float(model['std']) ** 2 * flip_energy(S), a2, J
