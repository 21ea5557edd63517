"""Acceptance checks for the predictor's virial (sgdml_b200_predict_virial, csrc/predict.cu): an FP64 oracle virial and a
componentwise bound.

With the rows r_i of a geometry and its cell L (lattice vectors as columns) strained homogeneously, r_i -> (I + eps) r_i
and L -> (I + eps) L, the virial is W = -dE/d(eps) at eps = 0.  E depends on the geometry only through x_d = 1/|delta_d|
(delta_d the minimum-image pair vector), and the oracle's descriptor-space force F_desc is -dE_raw/dx (F = std J^T F_desc
is -dE/dR), so
    W = -std sum_d F_desc[d] g_d delta_d^T,   g_d = delta_d / |delta_d|^3.
`oracle_virial` evaluates that from the oracle's own arrays (its permuted caches, alphas_E and descriptor code), with the
pair vectors and the image of oracle.desc.pbc_diff.  `strain_virial` is an independent estimate: central differences of
the oracle ENERGY under each of the six symmetric strains, Richardson-extrapolated.  `check_W` bounds |W - W_ref|
componentwise.  Plain functions on NumPy arrays, shared by tests/test_virial_checks.py (CPU) and
tests/test_predict_virial.py (GPU)."""

import copy

import numpy as np

import predict_checks as pc
from oracle import desc as odesc
from oracle import predict as opredict

U = pc.U


# ------------------------------------------------------------------------------------------------ models
def make_model(N, M, seed, ecstr=False, lattice=None, sig=20):
    """Random-coefficient model (std and c away from 1 and 0) on seeded synthetic training geometries, built with the
    oracle's descriptor code; ecstr: mixed-sign alphas_E; lattice: training descriptors and model in that cell."""
    from sgdml_b200 import synth

    perms = synth.rotor_swap_group(N, 1, 1)
    R = synth.geometries(N, M, seed).reshape(M, -1)
    rng = np.random.default_rng(seed + 99)
    alphas = rng.standard_normal(M * 3 * N)
    lat_and_inv = None if lattice is None else (lattice, np.linalg.inv(lattice))
    x, g = odesc.from_R(R, lat_and_inv)
    model = {
        'type': 'm',
        'z': np.ones(N, dtype=np.int64),
        'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(g, alphas.reshape(M, -1)),
        'alphas_F': alphas,
        'c': 0.37,
        'std': 1.7,
        'sig': sig,
        'lam': 1e-10,
        'perms': perms,
        'tril_perms_lin': odesc.tril_perms_lin(perms),
        'use_E': True,
    }
    if ecstr:
        model['alphas_E'] = 3.0 * rng.standard_normal(M)
    if lattice is not None:
        model['lattice'] = np.asarray(lattice, dtype=np.float64)
    return model


def queries(N, B, seed, lattice=None, margin=1e-6):
    """B seeded query geometries; in a cell, those within `margin` of a rounding tie (pc.pbc_margin) are skipped."""
    from sgdml_b200 import synth

    if lattice is None:
        return synth.geometries(N, B, seed).reshape(B, -1)
    R = synth.geometries(N, 2 * B, seed).reshape(2 * B, -1)
    keep = pc.pbc_margin(R, lattice, np.linalg.inv(lattice)) >= margin
    assert np.sum(keep) >= B
    return np.ascontiguousarray(R[keep][:B])


def with_cell(op, lattice):
    """A shallow copy of an oracle Predictor that builds its query descriptors in `lattice` (None: free molecule)."""
    q = copy.copy(op)
    q.lat_and_inv = None if lattice is None else (np.asarray(lattice, dtype=np.float64), np.linalg.inv(lattice))
    return q


# ------------------------------------------------------------------------------------------------ oracle virial
def pair_vectors(R, lat_and_inv):
    """Minimum-image pair vectors delta (B, D, 3), r_a - r_b in tril order with oracle.desc.pbc_diff's image."""
    R = np.asarray(R, dtype=np.float64)
    r = R.reshape(R.shape[0], -1, 3)
    a, b = odesc.tril_pairs(r.shape[1])
    d = r[:, a, :] - r[:, b, :]
    return d if lat_and_inv is None else odesc.pbc_diff(d, lat_and_inv)


def oracle_fdesc(op, r_desc):
    """The oracle's descriptor-space force of one query (oracle.predict.Predictor._raw, predict.py:199-229): unscaled,
    F = std J^T F_desc."""
    sig = op.sig
    diff = r_desc[None, :] - op.R_desc_perms
    norm = np.sqrt(5.0) * np.sqrt(np.sum(diff * diff, axis=1))
    base = np.exp(-norm / sig) * 5.0 / (3 * sig ** 3)
    a_x2 = np.einsum('ji,ji->j', diff, op.R_d_desc_alpha_perms)
    Fd = (a_x2 * base).dot(diff) * (5.0 / sig)
    base = base * (norm + sig)
    Fd -= base.dot(op.R_d_desc_alpha_perms)
    if op.alphas_E_lin is not None:
        Fd += op.alphas_E_lin.dot(diff * base[:, None])
    return Fd


def virial_from(Fd, g, delta, std):
    """W (B, 3, 3) = -std sum_d Fd[b, d] g[b, d] delta[b, d]^T."""
    return -std * np.einsum('bd,bdi,bdj->bij', Fd, g, delta)


def oracle_virial(op, R):
    """(E, F, W, Fd) of the oracle Predictor `op` (in its cell, op.lat_and_inv) for queries R (B, 3N)."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * op.n_atoms)
    x, g = odesc.from_R(R, op.lat_and_inv)
    Fd = np.array([oracle_fdesc(op, xi) for xi in x])
    W = virial_from(Fd, g, pair_vectors(R, op.lat_and_inv), op.std)
    E, F = op.predict(R)
    return E, F, W, Fd


def classical_virial(R, F):
    """sum_i r_i F_i^T (B, 3, 3)."""
    R = np.asarray(R, dtype=np.float64)
    B = R.shape[0]
    return np.einsum('bni,bnj->bij', R.reshape(B, -1, 3), np.asarray(F, dtype=np.float64).reshape(B, -1, 3))


STRAINS = [(0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1)]  # Voigt order


def strain_virial(op, R, h=1e-4):
    """W (B, 3, 3) from the oracle ENERGY alone: for each of the six symmetric strains eps = t (e_ij + e_ji) / 2 (e_ii
    on the diagonal), positions r -> (I + eps) r and the cell (when there is one) L -> (I + eps) L, central differences
    -dE/dt at steps h and h/2, Richardson-extrapolated: (4 D(h/2) - D(h)) / 3, error O(h^4)."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * op.n_atoms)
    B = R.shape[0]
    r = R.reshape(B, -1, 3)
    L = None if op.lat_and_inv is None else op.lat_and_inv[0]

    def energy(eps):
        A = np.eye(3) + eps
        q = with_cell(op, None if L is None else A @ L)
        return q.predict(np.einsum('ij,bnj->bni', A, r).reshape(B, -1))[0]

    W = np.empty((B, 3, 3))
    for i, j in STRAINS:
        e = np.zeros((3, 3))
        e[i, j] += 0.5
        e[j, i] += 0.5

        def dE(t):
            return (energy(t * e) - energy(-t * e)) / (2 * t)

        w = -(4 * dE(h / 2) - dE(h)) / 3
        W[:, i, j] = W[:, j, i] = w
    return W


# ------------------------------------------------------------------------------------------------ the bound
def fdesc_abs_scale(model, op, r_desc):
    """Componentwise magnitude of F_desc for one query: the F_desc of predict_checks.predict_abs_scale (before J^T),
    i.e. sum_k |c1_k| A_k + |c2_k| |JA_k| with the expanded-distance terms; see that docstring."""
    X = np.asarray(model['R_desc'], dtype=np.float64).T
    M = X.shape[0]
    mu = X.mean(axis=0)
    Xp = op.R_desc_perms
    mu_p = np.tile(op._perm_cache(mu[None]), (M, 1))
    xc = np.abs(Xp - mu_p)
    JAa = np.abs(op.R_d_desc_alpha_perms)
    JA2 = np.sqrt(np.sum(JAa * JAa, axis=1))
    ae = np.abs(op.alphas_E_lin) if op.alphas_E_lin is not None else None
    sig = op.sig
    diff = r_desc[None, :] - Xp
    norm = np.sqrt(5.0) * np.sqrt(np.sum(diff * diff, axis=1))
    base = np.exp(-norm / sig) * 5.0 / (3 * sig ** 3)
    qc = np.abs(r_desc[None, :] - mu_p)
    A = qc + xc
    rho = np.sum(qc * qc, axis=1) + np.sum(xc * xc, axis=1)
    a_abs = np.einsum('kd,kd->k', A, JAa)
    c2 = base * (norm + sig) + base * 5.0 * rho / sig
    c1 = a_abs * base * 5.0 / sig + base * (5.0 / sig) * 2 * np.sqrt(5.0) * JA2 * rho / sig
    if ae is not None:
        c1 = c1 + ae * c2
    return c1.dot(A) + c2.dot(JAa)


def virial_abs_scale(model, R, op=None):
    """(sW, bW), each (B, 3, 3), for check_W: sW = |std| sum_d |F_desc|_d |g_d| |delta_d|^T with |F_desc| from
    fdesc_abs_scale; bW = the pair-vector rounding of the wrap (zero for free molecules, see check_W)."""
    op = op if op is not None else opredict.Predictor(model)
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * op.n_atoms)
    x, g = odesc.from_R(R, op.lat_and_inv)
    delta = pair_vectors(R, op.lat_and_inv)
    FdA = np.array([fdesc_abs_scale(model, op, xi) for xi in x])
    std = abs(op.std)
    sW = std * np.einsum('bd,bdi,bdj->bij', FdA, np.abs(g), np.abs(delta))
    bW = np.zeros_like(sW)
    if op.lat_and_inv is not None:
        lat, lat_inv = op.lat_and_inv
        _, bg = pc.desc_pbc_bound(R, lat, lat_inv)
        Fd = np.array([oracle_fdesc(op, xi) for xi in x])
        dist = np.sqrt(np.sum(delta * delta, axis=-1))
        t = (np.abs(Fd) + FdA) * bg * dist
        bW += (WRAP_C * std * np.sum(t, axis=1))[:, None, None]
    return sW, bW


WRAP_C = 4 * np.sqrt(3.0)


def check_W(W, W_ref, scale, k, what='virial'):
    """|W - W_ref| <= tau(k) sW + bW componentwise, tau = pc.tau(k) = 8 k u (k = pc.n_terms(M, S, D)), scale = (sW, bW)
    from virial_abs_scale.  Returns max |W - W_ref| / sW for reporting.  A NaN fails.

    Derivation.  Both sides form W = -std sum_d F_desc[d] (g_d delta_d^T) with D pair terms.
      * F_desc: check_predict's derivation bounds each entry of the kernel's and the oracle's F_desc (the quantity before
        J^T) within gamma_{2M + D + S(sp+1) + 25} and gamma_{MS + D + 10} of its predict_abs_scale term, which is
        fdesc_abs_scale here; together below 6 k u (1 + O(ku)) of it for every tested shape (S >= 2 or M >= D + N + 40).
      * The pair factor: the engine rebuilds delta = g |g|^-3/2 from its g (|g|^2: 3 roundings, two square roots, the
        product, the division and the products g_i g_j s: 7 more, half of the square roots' errors), the oracle
        multiplies its g by its delta: within 10u of |g_i| |delta_j| each.
      * The sum over d: D terms, gamma_D; the std product: u.  These add (D + 12) u <= k u.
      The total stays below 7 k u of sW: c = 8 as in check_predict.
      * Cells: the two sides' g and delta differ by the rounding of the wrap itself, relative to |w| = |d| + |L||k| and
        not to |delta| (pc.desc_pbc_bound: |dg_c| <= bg = DESC_C u |w| / |delta|^3).  Through delta = g |g|^-3/2,
        |d delta| <= (1 + 3/2) |dg| |g|^-3/2 = 2.5 |dg| |delta|^3, so |d(g delta^T)_ij| <= |dg| |delta| + |g| |d delta|
        <= 3.5 |dg|_2 |delta| <= 4 sqrt(3) bg |delta|: bW = 4 sqrt(3) |std| sum_d (|F_desc_d| + |F_desc|_d) bg_d
        |delta_d|, the same for every entry.  The descriptor's own rounding moves F_desc by a relative DESC_C u |w| / |delta| times the Matern
        factors' n/sig, far below tau for the tested cells (|w| / |delta| < 10)."""
    sW, bW = scale
    W = np.asarray(W, dtype=np.float64).reshape(-1, 3, 3)
    W_ref = np.asarray(W_ref, dtype=np.float64).reshape(-1, 3, 3)
    err = np.abs(W - W_ref)
    bound = pc.tau(k) * sW + bW
    ok = err <= bound
    if not np.all(ok):
        bad = np.argwhere(~ok)
        i = tuple(int(j) for j in bad[0])
        raise AssertionError('%s: %d virial entries outside the bound; first at %s: |err| %r > %r'
                             % (what, bad.shape[0], i, float(err[i]), float(bound[i])))
    return float(np.max(err / sW))
