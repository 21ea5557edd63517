"""Test infrastructure for the Hessian-vector product (sgdml_b200_predict_hvp, torchtools.GDMLTorchPredict).

- `TorchOracle`: a float64 torch-on-CPU restatement of oracle.predict.Predictor._raw (descriptors, minimum image,
  energy constraints), differentiable end to end.  Its HV = (dF/dR) V comes from forward-mode autograd on F, so it
  is independent of the engine's hand-derived tangent formulas.
- `gemm_form_hvp`: a NumPy model of the engine's GEMM-composed HVP (csrc/predict.cu: stacked query and tangent rows,
  k_transform_tangent_rows with its floor under n, the permutation fold and k_tangent_project), run on the same GEMM-form
  quantities (S1 = Q Xc^T, ..., x5 = 5 (qq + mm) - 10 S1) that the device computes.
"""

import numpy as np
import torch

from oracle import desc as odesc
from oracle import predict as opredict

# csrc/predict.cu HVP_X5_FLOOR
X5_FLOOR = 5.0 * 64.0 * np.finfo(np.float64).eps


def _cell(model, lat_and_inv):
    """'model': the model's own cell (as oracle.predict.Predictor); None: a free molecule; else (lat, lat_inv)."""
    if isinstance(lat_and_inv, str):
        if 'lattice' not in model:
            return None
        lat = np.asarray(model['lattice'], dtype=np.float64)
        return lat, np.linalg.inv(lat)
    return lat_and_inv


FIXTURES = ['n5_m10_s1', 'n9_m16_s6', 'n12_m8_s12', 'n21_m6_s6', 'ecstr_n6_m8', 'pbc_n6_m8', 'big_n100_m2_s12']


def fixture_model(name):
    """(model, R_query, R_train (M, 3N)) of a golden fixture: its alphas_E or lattice when it has one; the files that
    keep only rows of the descriptor arrays (big_n240_m2_s3, big_n370_m2_s3) get them from oracle.desc."""
    from conftest import golden_model, load_golden

    g = load_golden(name)
    M = g['R_train'].shape[0]
    R_train = g['R_train'].reshape(M, -1)
    if 'model_R_desc' not in g:
        g['tril_perms_lin'] = odesc.tril_perms_lin(g['perms'])
        x, gd = odesc.from_R(R_train)
        g['model_R_desc'] = np.ascontiguousarray(x.T)
        g['R_d_desc_alpha'] = odesc.d_desc_dot_vec(gd, g['alphas_F'].reshape(M, -1))
    model = golden_model(g)
    if 'alphas_E' in g and g['alphas_E'].shape == (M,):
        model['alphas_E'] = g['alphas_E']
    if 'lattice' in g:
        model['lattice'] = g['lattice']
    return model, np.asarray(g['R_query'], dtype=np.float64), R_train


def signed_pairs(n_atoms):
    """P (D, N): +1 at atom b and -1 at atom a of pair d = (a, b), a > b, so that J^T w = P^T (g w) per component."""
    a, b = odesc.tril_pairs(n_atoms)
    P = np.zeros((len(a), n_atoms))
    P[np.arange(len(a)), b] = 1.0
    P[np.arange(len(a)), a] = -1.0
    return P


class TorchOracle(object):
    def __init__(self, model, lat_and_inv='model'):
        op = opredict.Predictor(model)
        self.n_atoms = op.n_atoms
        self.sig, self.std, self.c = op.sig, op.std, op.c
        self.cell = _cell(model, lat_and_inv)
        self.Xp = torch.from_numpy(np.ascontiguousarray(op.R_desc_perms, dtype=np.float64))
        self.JAp = torch.from_numpy(np.ascontiguousarray(op.R_d_desc_alpha_perms, dtype=np.float64))
        self.ae = None if op.alphas_E_lin is None else torch.from_numpy(op.alphas_E_lin)
        self.a, self.b = (torch.from_numpy(i) for i in odesc.tril_pairs(self.n_atoms))
        self.P = torch.from_numpy(signed_pairs(self.n_atoms))

    def ef(self, R):
        """R (B, 3N) float64 tensor -> E (B,), F (B, 3N), scaled as oracle.predict.Predictor.predict."""
        B, N = R.shape[0], self.n_atoms
        r = R.reshape(B, N, 3)
        pd = r[:, self.a] - r[:, self.b]
        if self.cell is not None:  # the image shift is locally constant
            lat, lat_inv = (torch.from_numpy(np.asarray(m, dtype=np.float64)) for m in self.cell)
            k = torch.round(torch.einsum('ij,bdj->bdi', lat_inv, pd.detach()))
            pd = pd - torch.einsum('ij,bdj->bdi', lat, k)
        dist = torch.sqrt((pd * pd).sum(-1))
        x = 1.0 / dist
        g = pd / (dist**3)[..., None]
        sig = self.sig
        diff = x[:, None, :] - self.Xp[None]
        norm = np.sqrt(5.0) * torch.sqrt((diff * diff).sum(-1))
        base = torch.exp(-norm / sig) * (5.0 / (3 * sig**3))
        a_x2 = torch.einsum('bkd,kd->bk', diff, self.JAp)
        Fd = torch.einsum('bk,bkd->bd', a_x2 * base, diff) * (5.0 / sig)
        base = base * (norm + sig)
        Fd = Fd - base @ self.JAp
        E = (a_x2 * base).sum(1)
        if self.ae is not None:
            Fd = Fd + torch.einsum('k,bk,bkd->bd', self.ae, base, diff)
            K_ee = (1 + (norm / sig) * (1 + norm / (3 * sig))) * torch.exp(-norm / sig)
            E = E + K_ee @ self.ae
        F = torch.einsum('dn,bdc->bnc', self.P, g * Fd[..., None]).reshape(B, 3 * N)
        return E * self.std + self.c, F * self.std

    def ef_np(self, R):
        with torch.no_grad():
            E, F = self.ef(torch.from_numpy(np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 3 * self.n_atoms)))
        return E.numpy(), F.numpy()

    def hvp(self, R, V):
        """(dF/dR) V by forward-mode autograd: NumPy (B, 3N) in and out."""
        R = torch.from_numpy(np.ascontiguousarray(R, dtype=np.float64).reshape(-1, 3 * self.n_atoms))
        V = torch.from_numpy(np.ascontiguousarray(V, dtype=np.float64).reshape(R.shape))
        _, HV = torch.func.jvp(lambda r: self.ef(r)[1], (R,), (V,))
        return HV.detach().numpy()

    def hessian(self, R):
        """dE^2/dR^2 = -dF/dR of one geometry R (3N,) -> (3N, 3N)."""
        R = torch.from_numpy(np.ascontiguousarray(R, dtype=np.float64).reshape(1, -1))
        J = torch.autograd.functional.jacobian(lambda r: self.ef(r)[1][0], R)
        return -J.reshape(R.shape[1], R.shape[1]).numpy()


def central_diff_hvp(f_of_R, R, V, h=1e-5):
    """(F(R + h V) - F(R - h V)) / 2h for a force function f_of_R: (B, 3N) -> (B, 3N)."""
    return (f_of_R(R + h * V) - f_of_R(R - h * V)) / (2 * h)


DEFECTS = ('dJ', 'csT', 'ae_dc2', 'pinv_fold')


def gemm_form_hvp(model, R, V, lat_and_inv='model', guard=True, defect=None, floor_scale=1.0):
    """The engine's HVP in NumPy, R, V (B, 3N) -> HV (B, 3N).  guard=False drops the floor under n in a ds / n and
    clamps x5 at 1e-300 as the forward does.  defect (for showing that a check fails; one of DEFECTS): 'dJ' drops the
    (dJ)^T F_desc term of k_tangent_project, 'csT' the (sum c1) T term of dG, 'ae_dc2' leaves ae dc2 out of dc1,
    'pinv_fold' folds the permutations with pinv instead of perm; floor_scale multiplies the floor."""
    assert defect is None or defect in DEFECTS, defect
    R = np.asarray(R, dtype=np.float64).reshape(-1, np.asarray(model['z']).shape[0] * 3)
    V = np.asarray(V, dtype=np.float64).reshape(R.shape)
    N = R.shape[1] // 3
    sig = float(model['sig'])
    std = float(model['std']) if 'std' in model else 1.0
    X = np.asarray(model['R_desc'], dtype=np.float64).T
    JA = np.asarray(model['R_d_desc_alpha'], dtype=np.float64)
    D = X.shape[1]
    mu = X.mean(0)
    Xc = X - mu
    S = int(np.asarray(model['perms']).shape[0])
    perm = odesc.tril_perms_from_lin(model['tril_perms_lin'], S)
    pinv = np.empty_like(perm)
    for p in range(S):
        pinv[p, perm[p]] = np.arange(D)
    ae = np.asarray(model['alphas_E'], dtype=np.float64) if 'alphas_E' in model else None
    mm = (Xc * Xc).sum(1)
    xja = (Xc * JA).sum(1)
    k_base = 5.0 / (3.0 * sig**3)
    k_c1 = k_base * 5.0 / sig
    xq, gq = odesc.from_R(R, _cell(model, lat_and_inv))
    t = odesc.d_desc_dot_vec(gq, V)
    P = signed_pairs(N)
    a_idx, b_idx = odesc.tril_pairs(N)
    out = np.empty_like(R)
    for i in range(R.shape[0]):
        Q = xq[i][pinv] - mu
        T = t[i][pinv]
        qq = (Q * Q).sum(1)[:, None]
        qt = (Q * T).sum(1)[:, None]
        S1, S2, S3, S4 = Q @ Xc.T, Q @ JA.T, T @ Xc.T, T @ JA.T
        a = S2 - xja
        x5 = 5.0 * (qq + mm) - 10.0 * S1
        n = np.sqrt(np.maximum(x5, 1e-300))
        e = np.exp(-n / sig)
        c2 = k_base * e * (n + sig)
        c1 = k_c1 * e * a
        ds = qt - S3
        floor = X5_FLOOR * floor_scale * (qq + mm) if guard else 0.0
        nf = np.sqrt(np.maximum(x5, np.maximum(floor, 1e-300)))
        dc2 = -5.0 * k_base * e * ds / sig
        dc1 = k_c1 * e * (S4 - 5.0 * a * ds / (nf * sig))
        if ae is not None:
            c1 = c1 + ae * c2
            if defect != 'ae_dc2':
                dc1 = dc1 + ae * dc2
        cs = c1.sum(1)[:, None]
        G = cs * Q - c1 @ Xc - c2 @ JA
        dG = dc1.sum(1)[:, None] * Q + (0.0 if defect == 'csT' else cs * T) - dc1 @ Xc - dc2 @ JA
        fold = pinv if defect == 'pinv_fold' else perm
        Fd = sum(G[p][fold[p]] for p in range(S))
        dFd = sum(dG[p][fold[p]] for p in range(S))
        g = gq[i]
        v = V[i].reshape(N, 3)
        dd = v[a_idx] - v[b_idx]
        gn = np.sqrt((g * g).sum(1))[:, None]
        dg = gn**1.5 * dd - 3.0 * (g * dd).sum(1)[:, None] * g / np.sqrt(gn)
        h = g * dFd[:, None] + (0.0 if defect == 'dJ' else dg * Fd[:, None])
        out[i] = std * (P.T @ h).ravel()
    return out
