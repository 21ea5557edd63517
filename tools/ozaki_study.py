"""CPU feasibility study (NumPy, exact integer arithmetic) for running the Cholesky trailing updates
of the analytic solve as FP64-via-INT8 GEMMs on the int8 tensor cores (Ozaki-style error-free
splitting): how many 7-bit slices does the sGDML system need so that the trained model still meets
the 1e-6 force tolerance?

For C -= W W^T every row of W is scaled by a power of two and cut into `s` signed 7-bit slices
(int8); every slice-pair product W_p W_q^T is an exact int32 GEMM (what `wgmma` s8 with a
int32 register accumulator computes), and the pairs with p + q <= s + 1 are summed in FP64.  The panel
work (potf2, TRSM) stays in FP64.  Nothing here is product code.

    python tools/ozaki_study.py [--n-atoms 21] [--n-train 40] [--nb 128]
"""
import argparse
import sys
import time

import numpy as np
import scipy.linalg

sys.path.insert(0, __file__.rsplit('/', 2)[0])
from oracle import assemble as oassemble  # noqa: E402
from oracle import desc as odesc  # noqa: E402
from oracle import predict as opredict  # noqa: E402
from sgdml_b200 import synth  # noqa: E402

BITS = 7


def split_rows(A, s):
    """A (m, k) -> exponents e (m,), slices (s, m, k) int64 with A ~= 2^e * sum_p slices[p] 2^(-BITS (p+1))."""
    amax = np.max(np.abs(A), axis=1)
    e = np.where(amax > 0, np.ceil(np.log2(np.where(amax > 0, amax, 1.0))) + 1, 0.0)  # |A| / 2^e < 1/2
    r = A / np.exp2(e)[:, None]
    # the slices are small integers; they are kept in float64 so that BLAS multiplies them -- exactly, since
    # every partial sum is an integer below 2^53 (|q| <= 64, k <= 2^17)
    out = np.empty((s,) + A.shape)
    for p in range(s):
        r = r * (1 << BITS)
        q = np.rint(r)  # round to nearest: |q| <= 64, remainder in [-1/2, 1/2]
        out[p] = q
        r = r - q
    return e, out


def ozaki_gemm_nt(A, B, s):
    """A B^T with s slices per operand; slice-pair products are exact integers."""
    ea, sa = split_rows(A, s)
    eb, sb = split_rows(B, s)
    C = np.zeros((A.shape[0], B.shape[0]))
    for level in range(2, s + 2):  # p + q (1-based) = level; smallest terms first would be better, keep it simple
        acc = np.zeros((A.shape[0], B.shape[0]))
        for p in range(1, level):
            q = level - p
            if p <= s and q <= s:
                acc += sa[p - 1] @ sb[q - 1].T  # exact integers (|entries| <= 64^2 k)
        C += acc * 2.0 ** (-BITS * level)
    return C * np.exp2(ea)[:, None] * np.exp2(eb)[None, :]


def blocked_cholesky(A, nb, gemm):
    """Right-looking blocked Cholesky (lower), trailing update through `gemm(W, W) -> W W^T`."""
    A = A.copy()
    n = A.shape[0]
    for j in range(0, n, nb):
        je = min(j + nb, n)
        A[j:je, j:je] = np.linalg.cholesky(A[j:je, j:je])
        if je < n:
            A[je:, j:je] = scipy.linalg.solve_triangular(A[j:je, j:je], A[je:, j:je].T, lower=True).T
            W = A[je:, j:je]
            A[je:, je:] -= gemm(W, W)
    return np.tril(A)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n-atoms', type=int, default=21)
    ap.add_argument('--n-train', type=int, default=40)
    ap.add_argument('--nb', type=int, default=128)
    ap.add_argument('--sig', type=float, default=20)
    ap.add_argument('--slices', default='4,5,6,7,8')
    a = ap.parse_args()
    N, M = a.n_atoms, a.n_train
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, a.sig)
    R = task['R_train'].reshape(M, -1)
    x, g = odesc.from_R(R)
    lin = odesc.tril_perms_lin(perms)
    t0 = time.time()
    K = oassemble.assemble(x, g, lin, a.sig, n_procs=8)
    n = K.shape[0]
    Amat = -K
    Amat[np.diag_indices(n)] += task['lam']
    y = task['F_train'].ravel().copy()
    std = np.std(y)
    y /= std
    print('n = %d, assembled in %.1f s, cond(-K + lam I) = %.2e' % (n, time.time() - t0, np.linalg.cond(Amat)))

    def model_for(alphas):
        return {'type': 'm', 'z': task['z'], 'R_desc': x.T, 'R_d_desc_alpha': odesc.d_desc_dot_vec(g, alphas.reshape(M, -1)),
                'alphas_F': alphas, 'c': 0.0, 'std': std, 'sig': a.sig, 'lam': task['lam'], 'perms': perms, 'tril_perms_lin': lin,
                'use_E': True}

    Rq = synth.geometries(N, 8, 1).reshape(8, -1)
    L_ref = blocked_cholesky(Amat, a.nb, lambda W, V: W @ V.T)
    al_ref = -scipy.linalg.cho_solve((L_ref, True), y)
    F_ref = opredict.Predictor(model_for(al_ref)).predict(Rq)[1]
    al_lapack = -scipy.linalg.cho_solve(scipy.linalg.cho_factor(Amat, lower=True), y)
    F_lapack = opredict.Predictor(model_for(al_lapack)).predict(Rq)[1]

    def rel(u, v):
        return float(np.max(np.abs(u - v)) / np.max(np.abs(v)))

    print('FP64 blocked vs LAPACK   : alphas %.2e  forces %.2e   (the noise floor of the problem)' % (rel(al_ref, al_lapack), rel(F_ref, F_lapack)))
    W = np.random.default_rng(0).standard_normal((256, a.nb))
    for s in [int(v) for v in a.slices.split(',')]:
        gerr = rel(ozaki_gemm_nt(W, W, s), W @ W.T)
        try:
            L = blocked_cholesky(Amat, a.nb, lambda W_, V_, s=s: ozaki_gemm_nt(W_, V_, s))
        except np.linalg.LinAlgError:
            print('s = %d: GEMM rel err %.1e, Cholesky breaks down (not positive definite)' % (s, gerr))
            continue
        al = -scipy.linalg.cho_solve((L, True), y)
        F = opredict.Predictor(model_for(al)).predict(Rq)[1]
        resid = np.linalg.norm(Amat @ (-al) - y) / np.linalg.norm(y)
        print('s = %d (%2d int8 GEMMs): GEMM rel err %.1e | alphas vs FP64 %.2e | forces vs FP64 %.2e | residual %.1e'
              % (s, s * (s + 1) // 2, gerr, rel(al, al_ref), rel(F, F_ref), resid))


if __name__ == '__main__' and not (len(sys.argv) > 1 and sys.argv[1] == 'predict'):
    main()


# ---------------------------------------------------------------------------------------------
# Second question: how many slices does the PREDICTOR need?  (python tools/ozaki_study.py predict)
def predict_gemm_form(model, R, gemm):
    """GEMM form of predict.py:199-217 as the engine evaluates it (permutations applied to the query:
    q_p[e] = x[pinv_p[e]]; descriptors centred by their column mean), with a pluggable A B^T."""
    N = len(model['z'])
    sig = float(model['sig'])
    S = len(np.asarray(model['perms']))
    D = N * (N - 1) // 2
    lin = np.asarray(model['tril_perms_lin']).reshape(D, S)  # lin[d*S + p] = perm_p[d] + p*D
    perm = (lin - np.arange(S)[None, :] * D).T  # (S, D): perm_p[d]
    pinv = np.argsort(perm, axis=1)
    X = np.asarray(model['R_desc']).T  # (M, D)
    JA = np.asarray(model['R_d_desc_alpha'])
    mu = X.mean(axis=0)
    Xc = X - mu
    xja = np.einsum('md,md->m', Xc, JA)
    mm = np.einsum('md,md->m', Xc, Xc)
    xq, gq = odesc.from_R(R)
    B = len(R)
    Q = np.stack([xq[b][pinv[p]] - mu for b in range(B) for p in range(S)])  # (B*S, D)
    qq = np.einsum('rd,rd->r', Q, Q)
    S1 = gemm(Q, Xc)
    S2 = gemm(Q, JA)
    n = np.sqrt(np.maximum(5.0 * (qq[:, None] + mm[None, :] - 2.0 * S1), 0.0))
    a = S2 - xja[None, :]
    e = np.exp(-n / sig)
    c1 = 25.0 / (3 * sig**4) * e * a
    c2 = 5.0 / (3 * sig**3) * (n + sig) * e
    G = c1.sum(axis=1)[:, None] * Q - gemm(c1, np.ascontiguousarray(Xc.T)) - gemm(c2, np.ascontiguousarray(JA.T))
    fd = np.zeros((B, D))
    for b in range(B):
        for p in range(S):
            fd[b] += G[b * S + p][perm[p]]
    return odesc.vec_dot_d_desc(gq, fd) * float(model['std'])


def main_predict():
    N, M = 21, 100
    perms = synth.rotor_swap_group(N, 1, 1)
    model = None
    from sgdml_b200 import synth as _s

    task = _s.make_task(N, M, perms, 20)
    R = task['R_train'].reshape(M, -1)
    x, g = odesc.from_R(R)
    lin = odesc.tril_perms_lin(perms)
    rng = np.random.default_rng(3)
    alphas = rng.standard_normal(M * 3 * N)
    model = {'type': 'm', 'z': task['z'], 'R_desc': x.T, 'R_d_desc_alpha': odesc.d_desc_dot_vec(g, alphas.reshape(M, -1)),
             'alphas_F': alphas, 'c': 0.0, 'std': 1.0, 'sig': 20, 'lam': 1e-10, 'perms': perms, 'tril_perms_lin': lin,
             'use_E': True}
    Rq = _s.geometries(N, 6, 1).reshape(6, -1)
    F_ref = opredict.Predictor(model).predict(Rq)[1]
    F64 = predict_gemm_form(model, Rq, lambda A, B: A @ B.T)
    print('GEMM form in FP64 vs direct form: %.2e' % (np.max(np.abs(F64 - F_ref)) / np.max(np.abs(F_ref))))
    for s in (3, 4, 5, 6, 7):
        F = predict_gemm_form(model, Rq, lambda A, B, s=s: ozaki_gemm_nt(A, B, s))
        print('S = %d (%2d int8 GEMMs): forces vs FP64 %.2e' % (s, s * (s + 1) // 2, np.max(np.abs(F - F_ref)) / np.max(np.abs(F_ref))))


if __name__ == '__main__' and len(sys.argv) > 1 and sys.argv[1] == 'predict':
    main_predict()
