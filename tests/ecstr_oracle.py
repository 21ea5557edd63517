"""Oracle (test infrastructure): the Nystroem-preconditioned CG of sgdml/solvers/iterative.py with energy
constraints in the kernel (use_E_cstr).

The system is (3NM + M)-square in the layout [forces; energies] (train.py:939-947): inducing columns index all
3NM + M columns (iterative.py:372-379), K_nm = assemble_E_cstr(...)[:, cols], K_mm = -K_nm[cols]
(iterative.py:232-253), and the operator returns [F; -E] - lam v (iterative.py:183-204).  The same restatement as
oracle/iterative.py, whose helpers (jitter escalation, preconditioner) it reuses.
"""

import numpy as np
import scipy as sp
import scipy.linalg
import scipy.sparse.linalg

from oracle import assemble as oassemble
from oracle import predict as opredict
from oracle.iterative import cho_factor_stable, precon


def nystroem_factor_ecstr(R_desc, R_d_desc, tril_perms_lin, sig, lam, col_idxs, force_qr=False):
    """B = L_inv_K_mn (m, 3NM + M), iterative.py:208-351 on the energy-constrained matrix.  force_qr: take the QR
    branch of iterative.py:312-322 even if the inner Cholesky factorisation would succeed (tests)."""
    col_idxs = np.asarray(col_idxs)
    K_nm = oassemble.assemble_E_cstr(R_desc, R_d_desc, tril_perms_lin, sig)[:, col_idxs]
    K_mm = -K_nm[col_idxs, :]
    L_mm, lower = cho_factor_stable(K_mm, pre_reg=True)
    K_nm = sp.linalg.solve_triangular(L_mm, K_nm.T, lower=lower, trans='T', check_finite=False).T
    inner = K_nm.T.dot(K_nm)
    inner[np.diag_indices_from(inner)] += lam
    res = None if force_qr else cho_factor_stable(inner, eps_mag_max=-14)
    if res is not None:
        L, lower = res
    else:
        m = K_nm.shape[1]
        L = np.linalg.qr(np.vstack([K_nm, np.sqrt(lam) * np.eye(m)]), mode='r')
        lower = False
    K_nm = sp.linalg.solve_triangular(L, K_nm.T, lower=lower, trans='T', check_finite=False).T
    return K_nm.T


def kernel_op_ecstr(model_like, R_desc, R_d_desc, lam):
    """iterative.py:183-204 with use_E_cstr: v = [v_F; v_E] -> [F; -E] - lam v of the oracle predictor with
    alphas_F = v_F, alphas_E = v_E (std = 1, c = 0)."""
    m = dict(model_like)
    m['std'], m['c'] = 1.0, 0.0
    n_train = R_desc.shape[0]
    m['alphas_E'] = np.zeros(n_train)
    p = opredict.Predictor(m)
    p.set_R_desc(R_desc)
    p.set_R_d_desc(R_d_desc)

    def K(v):
        p.set_alphas(v[:-n_train])
        # the oracle predictor keeps alphas_E repeated over the permutations (predict.py:443-447)
        p.alphas_E_lin = np.tile(np.asarray(v[-n_train:], dtype=np.float64)[:, None], (1, p.n_perms)).ravel()
        E, F = p.predict()
        return np.concatenate([F.ravel(), -E]) - lam * v

    return K


def solve_ecstr(model_like, R_desc, R_d_desc, tril_perms_lin, sig, lam, y, inducing_pts_idxs, tol=1e-4):
    """alphas = [alphas_F; alphas_E] via scipy.sparse.linalg.cg(-K_op, y, M=P_op, rtol=tol) (iterative.py:740-752)
    on the energy-constrained system; returns (alphas, info, iters, B)."""
    n = y.size
    B = nystroem_factor_ecstr(R_desc, R_d_desc, tril_perms_lin, sig, lam, inducing_pts_idxs)
    P = precon(B, lam)
    K = kernel_op_ecstr(model_like, R_desc, R_d_desc, lam)
    A_op = sp.sparse.linalg.LinearOperator((n, n), matvec=lambda v: -K(v))
    P_op = sp.sparse.linalg.LinearOperator((n, n), matvec=P)
    iters = [0]

    def cb(xk):
        iters[0] += 1

    x, info = sp.sparse.linalg.cg(A_op, y, M=P_op, rtol=tol, atol=0, maxiter=10 * n, callback=cb)
    return -x, info, iters[0], B
