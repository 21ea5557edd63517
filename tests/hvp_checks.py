"""Acceptance checks for the Hessian-vector product (sgdml_b200_predict_hvp): HV = (dF/dR) V against a long-double
reference with a componentwise bound.

Plain functions on NumPy arrays, shared by the GPU tests (tests/test_hvp_classes.py) and by a CPU test that shows the
reference is right and every check can fail (tests/test_hvp_checks.py).

- `hvp_reference` evaluates F and HV in np.longdouble with direct differences delta = q - x_{m,p} and the closed-form
  tangent formulas, valid on and near training points (the term (delta.JA)(delta.t)/|delta| has its exact limit 0).
- `hvp_abs_scale` and `check_hvp` give the componentwise bound |HV - HV_ref| <= tau(k) scale, in the style of
  predict_checks.predict_abs_scale / check_predict.
- `hvp_chunk_plan` restates how `sgdml_b200_predict_hvp` cuts a batch into chunks (tangent_plan with one direction).
"""

import collections

import numpy as np

import predict_checks as pc
from oracle import desc as odesc
from oracle import predict as opredict

U = pc.U
LD = np.longdouble
X5_FLOOR = 5.0 * 64.0 * np.finfo(np.float64).eps  # csrc/predict.cu HVP_X5_FLOOR
SQRT5 = np.sqrt(5.0)


def _require_long_double():
    """The reference is only a reference if it carries more bits than the FP64 it checks."""
    nmant = np.finfo(np.longdouble).nmant
    if nmant < 63:
        raise RuntimeError('np.longdouble has a %d-bit mantissa here: the HVP reference needs the 64-bit x87 format '
                           'and will not fall back to double' % nmant)


def _cell(model, lat_and_inv):
    """'model': the model's own cell (as oracle.predict.Predictor); None: a free molecule; else (lat, lat_inv)."""
    if isinstance(lat_and_inv, str):
        if 'lattice' not in model:
            return None
        lat = np.asarray(model['lattice'], dtype=np.float64)
        return lat, np.linalg.inv(lat)
    return lat_and_inv


class _Terms(object):
    """The model's training rows in the oracle's cache order, row k = m S + p (oracle.predict.Predictor): X_m and JA_m
    permuted by tril_perm_p, alphas_E repeated over the permutations."""

    def __init__(self, model, dtype):
        op = opredict.Predictor(model)
        self.N, self.S, self.M = op.n_atoms, op.n_perms, op.n_train
        self.D = self.N * (self.N - 1) // 2
        self.sig, self.std = op.sig, op.std
        self.Xp = op.R_desc_perms.astype(dtype)
        self.JAp = op.R_d_desc_alpha_perms.astype(dtype)
        self.ae = None if op.alphas_E_lin is None else op.alphas_E_lin.astype(dtype)
        X = np.asarray(model['R_desc'], dtype=np.float64).T
        self.mu_p = np.tile(op._perm_cache(X.mean(axis=0)[None]), (self.M, 1))  # engine's centring, permuted
        self.a, self.b = odesc.tril_pairs(self.N)


def _pair_vectors(R, N, cell, dtype):
    """Minimum-image pair vectors r_a - r_b (B, D, 3) in `dtype`.  The image k = round(lat_inv (r_a - r_b)) is taken
    in FP64 as oracle.desc.pbc_diff does (same images as the oracle), the shift L k is applied in `dtype`."""
    r = R.reshape(R.shape[0], N, 3)
    a, b = odesc.tril_pairs(N)
    pd = r[:, a, :] - r[:, b, :]
    if cell is not None:
        lat, lat_inv = (np.asarray(m, dtype=np.float64) for m in cell)
        k = np.around(np.einsum('ij,...j->...i', lat_inv, pd.astype(np.float64)))
        pd = pd - (lat.astype(dtype)[None, None] * k.astype(dtype)[:, :, None, :]).sum(-1)
    return pd


def _scatter_pairs(h, a, b, N):
    """P^T h per component: atom b gets +h_d, atom a gets -h_d (oracle.desc.vec_dot_d_desc) -> (3N,)."""
    out = np.zeros((N, 3), dtype=h.dtype)
    np.add.at(out, b, h)
    np.add.at(out, a, -h)
    return out.ravel()


def hvp_reference(model, R, V=None, lat_and_inv='model'):
    """F and HV = (dF/dR) V in np.longdouble: R, V (B, 3N) (FP64 or long double) -> (F, HV), both (B, 3N) long double
    (HV is None when V is None).

    Per geometry, with x, g = delta_pair / |delta_pair|^3 the descriptor and its Jacobian factor, t = J V, and for each
    cache row k (training point m, permutation p): delta = x - X_k, n = sqrt5 |delta|, e = exp(-n / sig),
    a = delta . JA_k, ds = delta . t (direct differences, never the GEMM expansion):
      c2 = k_base e (n + sig),   c1 = k_c1 e a + ae c2,      F_desc  = sum_k c1 delta - c2 JA_k
      dc2 = -5 k_base e ds / sig,   dc1 = k_c1 e (JA_k . t - 5 (a ds / n) / sig) + ae dc2
      dF_desc = sum_k dc1 delta + c1 t - dc2 JA_k
      F = std P^T (g F_desc),   HV = std P^T (g dF_desc + dg F_desc),
      dg = dd / |d|^3 - 3 (d . dd) d / |d|^5  (d the minimum-image pair vector, dd = v_a - v_b),
    with a ds / n = (delta.JA)(delta.t) / (sqrt5 |delta|) <= |JA| |t| |delta| / sqrt5 set to its limit 0 at delta = 0.
    The torch oracle's forward-mode sqrt is NaN there; this form is exact on and near training points."""
    _require_long_double()
    m = _Terms(model, LD)
    N, sig = m.N, LD(m.sig)
    cell = _cell(model, lat_and_inv)
    R = np.asarray(R)
    R = R.astype(LD).reshape(-1, 3 * N)
    pd = _pair_vectors(R, N, cell, LD)
    dist = np.sqrt((pd * pd).sum(-1))
    x = 1 / dist
    g = pd / (dist ** 3)[..., None]
    if V is not None:
        V = np.asarray(V).astype(LD).reshape(R.shape)
    k_base = LD(5) / (3 * sig ** 3)
    k_c1 = k_base * 5 / sig
    s5 = np.sqrt(LD(5))
    B = R.shape[0]
    F = np.empty((B, 3 * N), dtype=LD)
    HV = None if V is None else np.empty((B, 3 * N), dtype=LD)
    for i in range(B):
        delta = x[i][None, :] - m.Xp
        dl = np.sqrt((delta * delta).sum(1))
        n = s5 * dl
        e = np.exp(-n / sig)
        a = (delta * m.JAp).sum(1)
        c2 = k_base * e * (n + sig)
        c1 = k_c1 * e * a
        if m.ae is not None:
            c1 = c1 + m.ae * c2
        Fd = (c1[:, None] * delta).sum(0) - (c2[:, None] * m.JAp).sum(0)
        F[i] = _scatter_pairs(g[i] * Fd[:, None], m.a, m.b, N)
        if V is None:
            continue
        v = V[i].reshape(N, 3)
        dd = v[m.a] - v[m.b]
        t = -(g[i] * dd).sum(-1)
        ds = (delta * t[None, :]).sum(1)
        ads_n = np.zeros_like(dl)
        nz = dl > 0
        ads_n[nz] = a[nz] * ds[nz] / n[nz]
        dc2 = -5 * k_base * e * ds / sig
        dc1 = k_c1 * e * ((m.JAp * t[None, :]).sum(1) - 5 * ads_n / sig)
        if m.ae is not None:
            dc1 = dc1 + m.ae * dc2
        dFd = (dc1[:, None] * delta).sum(0) + c1.sum() * t - (dc2[:, None] * m.JAp).sum(0)
        d, d2 = pd[i], dist[i] ** 2
        dg = dd / (dist[i] ** 3)[:, None] - 3 * ((d * dd).sum(-1) / (d2 * d2 * dist[i]))[:, None] * d
        HV[i] = _scatter_pairs(g[i] * dFd[:, None] + dg * Fd[:, None], m.a, m.b, N)
    std = LD(m.std)
    return F * std, (None if HV is None else HV * std)


# ------------------------------------------------------------------------------------------------ magnitude
def hvp_abs_scale(model, R, V, lat_and_inv='model'):
    """Per-output magnitudes scale (B, 3N) for `check_hvp`: the engine's HVP (csrc/predict.cu,
    k_transform_tangent_rows, k_combine_tangent_rows, k_tangent_project) with every term replaced by its absolute value, so
    that tau(k) scale bounds the rounding of each term.  Notation per cache row k: q = x - mu and X_k - mu the centred
    query and training descriptors as the engine stores them, A = |q| + |X_k - mu| (componentwise), rho = |q|^2 +
    |X_k - mu|^2, ta_d = sum_c |g_dc| (|v_ac| + |v_bc|) (a bound on |t_d| and on its rounding), |.|_2 Euclidean norms.

      |a| -> A.|JA_k|,  |ds| -> A.ta,  |da| -> ta.|JA_k|      (a = S2 - xja and ds = qt - S3 are differences of
                                                              GEMM dot products: their rounding scales with |q| + |x|)
      erel = 1 + sqrt5 rho / (sig d_eff)                     (e's error through n, on the one term that is not
                                                              small near delta = 0, da; see check_hvp)
      |a ds / n| -> (A.|JA| |t|_2 + |JA|_2 A.ta + |JA|_2 |t|_2 rho / d_eff) / sqrt5 + |JA|_2 |t|_2 rho / sig
      c2 -> k_base e ((n + sig) + 5 rho / sig),  c1 -> k_c1 e (|a| + 2 sqrt5 |JA|_2 rho / sig) + |ae| c2
      dc2 -> 5 k_base e (|ds| + 2 sqrt5 |t|_2 rho / sig) / sig,  dc1 -> k_c1 e (erel |da| + 5 |a ds / n| / sig) + |ae| dc2
    (the rho / sig terms are e's error through n times |a| <= |delta| |JA|_2, |ds| <= |delta| |t|_2 and
    |a ds / n| <= |delta| |JA|_2 |t|_2 / sqrt5, as in predict_checks.predict_abs_scale; c2 is flat in n)
      F_desc -> sum_k c1 A + c2 |JA_k|,  dF_desc -> sum_k dc1 A + (sum_k c1) ta + dc2 |JA_k|
      HV -> |std| |P|^T (|g| dF_desc + dg F_desc),  dg_c = |g|_2^3/2 |dd_c| + 3 (|g|.|dd|) |g_c| / |g|_2^1/2
    with d_eff = 8 sqrt(u rho) (n_floor / sqrt5, the floor of the engine) where |delta| <= sqrt((4 D + 76) u rho), and
    |delta| elsewhere."""
    m = _Terms(model, np.float64)
    N, sig, D = m.N, m.sig, m.D
    cell = _cell(model, lat_and_inv)
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * N)
    V = np.asarray(V, dtype=np.float64).reshape(R.shape)
    xq, gq = odesc.from_R(R, cell)
    k_base = 5.0 / (3.0 * sig ** 3)
    k_c1 = k_base * 5.0 / sig
    xc = np.abs(m.Xp - m.mu_p)
    xc2 = (xc * xc).sum(1)
    JAa = np.abs(m.JAp)
    JA2 = np.sqrt((JAa * JAa).sum(1))
    ae = None if m.ae is None else np.abs(m.ae)
    out = np.empty_like(R)
    for i in range(R.shape[0]):
        g = np.abs(gq[i])
        v = np.abs(V[i].reshape(N, 3))
        dd = v[m.a] + v[m.b]
        ta = (g * dd).sum(-1)
        ta2 = np.sqrt((ta * ta).sum())
        qc = np.abs(xq[i][None, :] - m.mu_p)
        A = qc + xc
        rho = (qc * qc).sum(1) + xc2
        delta = xq[i][None, :] - m.Xp
        dl = np.sqrt((delta * delta).sum(1))
        d_eff = np.where(dl * dl <= (4 * D + 76) * U * rho, np.sqrt(64 * U * rho), dl)
        n = SQRT5 * dl
        e = np.exp(-n / sig)
        erel = 1.0 + SQRT5 * rho / (sig * d_eff)
        a_abs = (A * JAa).sum(1)
        ds_abs = A @ ta
        da_abs = JAa @ ta
        ads = (a_abs * ta2 + JA2 * ds_abs + JA2 * ta2 * rho / d_eff) / SQRT5 + JA2 * ta2 * rho / sig
        c2 = k_base * e * ((n + sig) + 5.0 * rho / sig)
        c1 = k_c1 * e * (a_abs + 2 * SQRT5 * JA2 * rho / sig)
        dc2 = 5.0 * k_base * e * (ds_abs + 2 * SQRT5 * ta2 * rho / sig) / sig
        dc1 = k_c1 * e * (erel * da_abs + 5.0 * ads / sig)
        if ae is not None:
            c1 = c1 + ae * c2
            dc1 = dc1 + ae * dc2
        Fd = c1 @ A + c2 @ JAa
        dFd = dc1 @ A + c1.sum() * ta + dc2 @ JAa
        gn = np.sqrt((g * g).sum(-1))
        dg = gn[:, None] ** 1.5 * dd + 3.0 * ((g * dd).sum(-1) / np.sqrt(gn))[:, None] * g
        h = g * dFd[:, None] + dg * Fd[:, None]
        o = np.zeros((N, 3))
        np.add.at(o, m.a, h)
        np.add.at(o, m.b, h)
        out[i] = o.ravel()
    return out * abs(m.std)


# ------------------------------------------------------------------------------------------------ the check
def n_terms(M, S, D, N):
    """k of the bound: the M S (training point, permutation) terms, the descriptor length and the atoms."""
    return M * S + D + N


def check_hvp(HV, HV_ref, scale, k, what='hvp'):
    """|HV - HV_ref| <= tau(k) scale componentwise, tau = c k u with c = predict_checks.CHECK_C = 8 and k = n_terms.
    Returns (max |HV - HV_ref| / scale, max(tau scale) / max |HV_ref|): the worst error in units of the scale, and the
    bound's tightness relative to the output.

    Derivation (u = 2^-53, gamma_n = n u / (1 - n u); each error is relative to the matching term of hvp_abs_scale,
    whose terms dominate the absolute values of everything the engine and the reference add up):
      * GEMM1 and the row dot products: S1..S4, qq, mm, xja, qt within gamma_D of their absolute sums, so a, ds and
        da = S4 are within gamma_{D+1} of A.|JA|, A.ta and ta.|JA| (the centring q = x - mu, X - mu cancels mu's own
        rounding and adds u A; t = J V is within gamma_4 ta).  x5 = 5 (qq + mm) - 10 S1 is within
        dx5 = 10 gamma_{D+2} rho of 5 |delta|^2.
      * e through n.  Away from a training point (|delta|^2 > (4 D + 76) u rho, so dx5 <= x5 / 2):
        |dn| <= n dx5 / x5 <= sqrt5 gamma_{D+2} rho / |delta| and e moves by e |dn| / sig <= gamma_{D+2} e (erel - 1);
        exp_neg and the rsqrt add <= 15 u.  Closer, |dn| <= sqrt(dx5) <= sqrt(10 (D+2) u rho), which is below
        k u sqrt5 rho / d_eff = k sqrt5 sqrt(u rho) when k^2 >= 2 (D + 2).
      * The a ds / n term (not (|q| + |x|)^2 / n: that is vacuous as n -> 0).  |a| <= |delta| |JA|_2 and |ds| <=
        |delta| |t|_2 bound the term by |delta| |JA|_2 |t|_2 / sqrt5, and its rounding stays bounded as n -> 0:
        da ds / n <= gamma A.|JA| |t|_2 / sqrt5, a d(ds) / n <= gamma |JA|_2 A.ta / sqrt5, and through n (relative
        error <= 2 gamma rho / |delta|^2 away from a training point) <= 2 gamma |JA|_2 |t|_2 rho / (sqrt5 |delta|) --
        the three parts of |a ds / n| in the scale.
      * The floor.  k_transform_tangent_rows divides by n_f = sqrt(max(x5, 320 u rho)) >= sqrt5 8 sqrt(u rho).  Where
        |delta|^2 <= (4 D + 76) u rho the floor may bite; there the engine's term is at most
        (|delta| |JA|_2 + da)(|delta| |t|_2 + d(ds)) / n_f ~ (4 D + 76) u rho |JA|_2 |t|_2 / (8 sqrt5 sqrt(u rho)) and
        the true one at most |delta| |JA|_2 |t|_2 / sqrt5, so the floor's replacement error is at most
        k_c1 e |JA_m|_2 |t|_2 n_floor / sig times (D / 2 + 10) / 8 -- and tau |JA|_2 |t|_2 rho / (sqrt5 d_eff) with
        d_eff = 8 sqrt(u rho) is k sqrt(u rho) |JA|_2 |t|_2 / sqrt5: enough when 8 k >= 4 D + 76.
      * GEMM2 sums 2 M + 1 terms per virtual row (padded training columns are zero: exact), k_combine_tangent_rows
        two roundings, the fold over S permutations S, k_tangent_project N - 1 pairs of <= 4 roundings each.  It rebuilds
        the pair vector from g (|g|_2 = |d|^-2, 3 + 2 roundings), so dg carries <= 10 u of the dg of the scale; the
        difference dF_desc - 3 (g.dd) F_desc / |g|^1/2 is bounded by the sum of absolute values.  std: one rounding.
    The engine's error is therefore within gamma_{3 D + 2 M + S + 4 N + 40} of the scale, and the reference's (long
    double, u_ld = u / 2048, with the same sums over M S rows, D entries and N atoms) within gamma_k / 1000.  Both are
    below 4 k u for every shape the tests use (S >= 2, or M >= D), so c = 8 leaves a margin of 2.
    Query descriptors carry a few u of |x| (more behind a cell's image shift, a factor |w| / |d'| as in
    predict_checks.desc_pbc_bound); the margin absorbs it.  A NaN anywhere fails the check (NaN <= bound is false)."""
    t = pc.tau(k)
    HV = np.asarray(HV, dtype=np.float64)
    HV_ref = np.asarray(HV_ref, dtype=np.float64)
    scale = np.asarray(scale, dtype=np.float64)
    err = np.abs(HV - HV_ref)
    ok = err <= t * scale
    if not np.all(ok):
        bad = np.argwhere(~ok)
        i = tuple(int(j) for j in bad[0])
        raise AssertionError('%s: %d HV entries outside tau = %.2e times the scale; first at %s: |err| %r > %r '
                             '(|err|/scale %.2e)' % (what, bad.shape[0], t, i, float(err[i]), float(t * scale[i]),
                                                     float(err[i] / scale[i])))
    ratio = float(np.max(err / scale)) if err.size else 0.0
    tight = float(t * np.max(scale) / max(np.max(np.abs(HV_ref)), 1e-300)) if err.size else 0.0
    return ratio, tight


def check_against_reference(HV, model, R, V, what='hvp', lat_and_inv='model'):
    """check_hvp of HV against hvp_reference with hvp_abs_scale and n_terms of the model: (ratio, tightness)."""
    _, ref = hvp_reference(model, R, V, lat_and_inv)
    scale = hvp_abs_scale(model, R, V, lat_and_inv)
    return check_hvp(HV, ref, scale, model_terms(model), what)


# ------------------------------------------------------------------------------------------------ models
SIG = 20
# name: (N, M) -- one per padded descriptor width DP of the fused classes, D just past 256 (N = 24, GEMM form) and
# D = 435; M is one more than a multiple of the class's BM, so Mpad > M and padded training columns are exercised
CLASSES = {
    'dp40': (9, 33),
    'dp72': (12, 33),
    'dp112': (15, 33),
    'dp160': (18, 33),
    'dp224': (21, 33),
    'dp256': (23, 25),
    'n24': (24, 25),
    'n30': (30, 17),
}
VARIANTS = ('plain', 'ecstr', 'pbc')
PBC_MARGIN = 1e-6


def build_model(R_train, alphas_F, perms, sig=SIG, alphas_E=None, lattice=None):
    """A model dict from training geometries (M, 3N) and force coefficients, with std and c away from 1 and 0, optional
    alphas_E and a cell (training descriptors built in it)."""
    R_train = np.asarray(R_train, dtype=np.float64)
    M = R_train.shape[0]
    cell = None if lattice is None else (lattice, np.linalg.inv(lattice))
    x, g = odesc.from_R(R_train, cell)
    perms = np.asarray(perms, dtype=np.int64)
    model = {
        'type': 'm',
        'z': np.ones(R_train.shape[1] // 3, dtype=np.int64),
        'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(g, np.asarray(alphas_F).reshape(M, -1)),
        'alphas_F': np.asarray(alphas_F, dtype=np.float64),
        'c': 0.37,
        'std': 1.7,
        'sig': sig,
        'lam': 1e-10,
        'perms': perms,
        'tril_perms_lin': odesc.tril_perms_lin(perms),
        'use_E': True,
    }
    if alphas_E is not None:
        model['alphas_E'] = np.asarray(alphas_E, dtype=np.float64)
    if lattice is not None:
        model['lattice'] = np.asarray(lattice, dtype=np.float64)
    return model


def class_model(name, variant, seed=0):
    """(model, R_train) of a CLASSES shape (or the golden fixture big_n240_m2_s3): 'plain', 'ecstr' (seeded alphas_E
    large enough to move HV by well over 10 %) or 'pbc' (predict_checks.skewed_cell)."""
    from sgdml_b200 import synth

    rng = np.random.default_rng(seed + 99)
    if name == 'big_n240_m2_s3':
        from conftest import load_golden

        gd = load_golden(name)
        M = gd['R_train'].shape[0]
        R_train, alphas, perms, sig = gd['R_train'].reshape(M, -1), gd['alphas_F'], gd['perms'], int(gd['sig'])
        N = R_train.shape[1] // 3
    else:
        N, M = CLASSES[name]
        perms = synth.rotor_swap_group(N, 1, 1)
        R_train = synth.geometries(N, M, seed).reshape(M, -1)
        alphas, sig = rng.standard_normal(M * 3 * N), SIG
    ae = 3.0 * rng.standard_normal(M) if variant == 'ecstr' else None
    lattice = pc.skewed_cell(N) if variant == 'pbc' else None
    return build_model(R_train, alphas, perms, sig, ae, lattice), R_train


def queries(model, B, seed):
    """B seeded query geometries (and tangents V) of the model; in a cell, those within PBC_MARGIN of a rounding tie
    are replaced (few are)."""
    from sgdml_b200 import synth

    N = int(np.asarray(model['z']).shape[0])
    R = synth.geometries(N, 2 * B, seed).reshape(2 * B, -1)
    if 'lattice' in model:
        lat = np.asarray(model['lattice'])
        keep = pc.pbc_margin(R, lat, np.linalg.inv(lat)) >= PBC_MARGIN
        assert np.sum(~keep[:B]) <= max(2, B // 20), 'too many queries near a rounding tie'
        R = R[keep]
    R = np.ascontiguousarray(R[:B])
    return R, np.random.default_rng(seed + 7).standard_normal(R.shape)


def near_training(R_train, eps, seed):
    """Training geometries moved by eps (Angstrom, Euclidean norm over the geometry) along seeded random directions."""
    W = np.random.default_rng(seed).standard_normal(R_train.shape)
    return R_train + eps * W / np.linalg.norm(W, axis=1, keepdims=True)


def model_terms(model):
    """n_terms of a model dict."""
    N = int(np.asarray(model['z']).shape[0])
    return n_terms(int(np.asarray(model['R_desc']).shape[1]), int(np.asarray(model['perms']).shape[0]),
                   N * (N - 1) // 2, N)


# ------------------------------------------------------------------------------------------------ chunk plan
HvpPlan = collections.namedtuple('HvpPlan', 'chunk chunks edges')


def hvp_chunk_geos(layout, S, cap=0):
    """Geometries per HVP chunk (csrc/predict.cu tangent_plan with one direction per geometry): a stacked row holds
    DS + 2 Mpad + DP + 2 doubles (Qg, SX, SJ, G, qq, csum), a geometry 2 S rows (S query rows, S tangent rows), within
    2 GiB; at least 1, at most 65 536, at most `cap` (a cap of 2 cap S rows) when the test hook sets one."""
    DS = layout.DP + 4  # the model's row stride (m->DS in csrc/predict.cu); pc.Layout does not carry it
    rows = (2048 << 20) // (8 * (DS + 2 * layout.Mpad + layout.DP + 2))
    if cap > 0:
        rows = min(rows, 2 * cap * S)
    rows = max(rows, 2 * S)
    return min(rows // (2 * S), 65536)


def hvp_chunk_plan(layout, S, B, cap=0):
    """How `sgdml_b200_predict_hvp` runs B geometries: an HvpPlan of the chunk size, the [(lo, hi)] geometry ranges in
    launch order, and the edge rows (first and last geometry of every chunk)."""
    chunk = hvp_chunk_geos(layout, S, cap)
    chunks = [(lo, min(lo + chunk, B)) for lo in range(0, B, chunk)]
    return HvpPlan(chunk, chunks, sorted({r for lo, hi in chunks for r in (lo, hi - 1)}))
