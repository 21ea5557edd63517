"""Acceptance checks for the predictor (csrc/predict.cu): energies and forces against the oracle.

Plain functions on NumPy arrays, shared by the GPU tests (tests/test_predict_bulk.py) and by a CPU test that shows
every check can fail (tests/test_predict_checks.py).  Each check raises AssertionError with a short diagnosis.

`chunk_plan` restates how `sgdml_b200_predict` / `sgdml_b200_predict_train` cut a batch into chunks, so that the tests
know which rows sit on chunk edges and how many main-kernel launches the engine must count.  `main_schedule` restates
how one launch of the fused main kernel spreads its query tiles over persistent CTAs, so that the tests know which
rows each CTA computes in which sweep.  `predict_abs_scale` and `check_predict` give a componentwise error bound for E
and F.
"""

import collections
import math

import numpy as np

U = 2.0 ** -53

# ------------------------------------------------------------------------------------------------ chunk plan
# template arguments of the fused predictor's tile classes (csrc/predict.cu, the PCfg of each Cfg*), by padded
# descriptor length DP: (BQ, BM, W1Q, W1M, W1K, W2Q, W2D, MINB, W2S, OB)
PCFG = {
    40: (64, 32, 4, 2, 1, 4, 1, 2, 2, 0),
    72: (64, 32, 4, 2, 1, 4, 1, 1, 2, 1),
    112: (64, 16, 4, 2, 1, 4, 2, 1, 1, 1),
    160: (32, 16, 2, 2, 2, 2, 4, 1, 1, 1),
    224: (32, 16, 2, 2, 2, 2, 4, 1, 1, 1),
    256: (32, 8, 2, 1, 4, 2, 4, 1, 1, 0),
}
# (DP, BQ, BM) in kCfgs order; D > 256 runs the GEMM-composed path
_CFGS = tuple((DP, c[0], c[1]) for DP, c in sorted(PCFG.items()))
GRAPH_MAX_GEO = 16  # host-buffer batches up to this size replay a captured CUDA graph
PIPELINE_MIN_GEO = 4096  # host-buffer batches from this size run on two side streams

Layout = collections.namedtuple('Layout', 'D DP BQ BM Mpad large')
Plan = collections.namedtuple('Plan', 'chunks slots pipelined graph main_launches')


def layout(n_atoms, n_train):
    """The engine's padded model layout for N atoms and M training points (sgdml_b200_model_create)."""
    D = n_atoms * (n_atoms - 1) // 2
    for DP, BQ, BM in _CFGS:
        if D <= DP:
            return Layout(D, DP, BQ, BM, -(-n_train // BM) * BM, False)
    DP = -(-D // 8) * 8
    return Layout(D, DP, 8, 8, -(-n_train // 8) * 8, True)


def chunk_geos(DP, Mpad, S, large, cap=0):
    """Queries per chunk: G (rows x DP doubles) within 256 MB, or for D > 256 each of G and S1 / S2 (rows x Mpad) within
    2 GB; at least 1, at most 65 536, at most `cap` when the test hook sets one."""
    rows = (256 << 20) // (DP * 8)
    if large:
        rows = min((2048 << 20) // (DP * 8), (2048 << 20) // (Mpad * 8))
    g = min(max(rows // S, 1), 65536)
    return min(g, cap) if cap > 0 else g


def chunk_plan(D, DP, Mpad, S, large, B, host_io, cap=0, train=False):
    """How the engine runs a batch of B queries.

    host_io: R, E and F are all host buffers (NumPy arrays or host tensors).  train: `sgdml_b200_predict_train` over B
    training points (always one stream, no graph).  Returns a Plan:
      chunks       [(lo, hi)] query ranges, in launch order
      slots        workspace slot of each chunk (the pipeline alternates 0 / 1; otherwise 0)
      pipelined    chunks run on the two side streams (host buffers, B >= 4096)
      graph        the batch replays a captured CUDA graph as one piece (host buffers, B <= 16)
      main_launches  increment of the `predict_main` launch counter: one per chunk on the fused path (D <= 256), two per
                   chunk on the GEMM-composed path.  A graph replay counts its kernels under `predict_aux` only, so 0;
                   the first call at a new batch size launches twice (once plain, once under capture).
    D is the unpadded descriptor length (the plan depends on it only through DP and `large`)."""
    assert large == (D > 256)
    per_chunk = 2 if large else 1
    if B == 0:
        return Plan([], [], False, False, 0)
    if host_io and not train and B <= GRAPH_MAX_GEO:
        return Plan([(0, B)], [0], False, True, 0)
    chunk = min(chunk_geos(DP, Mpad, S, large, cap), B)
    pipelined = host_io and not train and B >= PIPELINE_MIN_GEO
    if pipelined:
        chunk = min(chunk, max(1024, (B + 3) // 4))
    chunks = [(lo, min(lo + chunk, B)) for lo in range(0, B, chunk)]
    slots = [(i & 1) if pipelined else 0 for i in range(len(chunks))]
    return Plan(chunks, slots, pipelined, False, per_chunk * len(chunks))


def edge_rows(plan):
    """First and last query of every chunk."""
    return sorted({r for lo, hi in plan.chunks for r in (lo, hi - 1)})


# ------------------------------------------------------------------------------------------------ main-kernel schedule
SM_SMEM = 228 * 1024  # shared memory per SM (H100)
CTA_SMEM_RESERVED = 1024  # reserved by the system per resident CTA
SM_THREADS = 2048
NT = 256  # threads per CTA of k_predict_main

Schedule = collections.namedtuple('Schedule', 'B S BQ q_tiles n_tiles n_splits tiles_per_split grid per_sm cta_tiles')


def smem_bytes(DP):
    """Dynamic shared memory of k_predict_main for the tile class of DP: PCfg's carve-up (SMEM_BYTES), in doubles
    Q [BQ DS], Xc and JA [2][BM DS] each, mm / xja / ae [2][BM] each, the S / C tiles [OB ? 2 : 1][PK][2][BQ CS],
    qq / csum / E [BQ] each, the XK exchange area and three mbarriers (4 doubles)."""
    BQ, BM, W1Q, W1M, W1K, W2Q, W2D, MINB, W2S, OB = PCFG[DP]
    DS, CS = DP + 4, BM + 4
    XK = bool(OB) and W1K == 2
    PK = 1 if XK else W1K
    n = BQ * DS + 2 * (2 * BM * DS) + 3 * (2 * BM) + (2 if OB else 1) * PK * 2 * BQ * CS + 3 * BQ
    n += (4 * 2 * 2 * 32 * 2 if XK else 0) + 4
    return 8 * n


def ctas_per_sm(DP):
    """Resident CTAs of the class on one SM as its shared memory allows (256 threads each; no class is held to fewer
    by its registers than by its shared memory)."""
    return min(SM_SMEM // (smem_bytes(DP) + CTA_SMEM_RESERVED), SM_THREADS // NT)


def main_schedule(N, M, S, B, n_sms, ws_geo=None):
    """How one launch of k_predict_main runs B geometries (B S virtual rows (b, p)) on a GPU of n_sms SMs
    (run_queries and launch_main_t in csrc/predict.cu):
      q_tiles = ceil(B S / BQ) query tiles, n_tiles = Mpad / BM training tiles;
      sp = ceil(2 n_sms / q_tiles), capped at the workspace rows over the batch's (ws_geo: the geometries the
           workspace slot holds; None leaves this cap out -- it cannot matter when sp is 1 anyway), at
           2 ceil(sqrt(2 n_tiles)) and at n_tiles, at least 1; the sweep is cut into n_splits = ceil(n_tiles / tps)
           pieces of tps = ceil(n_tiles / sp) tiles;
      grid = q_tiles with a split sweep or for the two-CTA class, otherwise min(q_tiles, n_sms per_sm) persistent CTAs;
      CTA x runs query tiles x, x + grid, ... (cta_tiles[x]), one sweep over its training tiles each.
    sp = 1 whatever the workspace when q_tiles >= 2 n_sms or n_tiles == 1."""
    ly = layout(N, M)
    assert not ly.large, 'the GEMM-composed path has no persistent main kernel'
    BQ, BM = ly.BQ, ly.BM
    MINB = PCFG[ly.DP][7]
    q_tiles = -(-B * S // BQ)
    n_rows_pad = q_tiles * BQ
    n_tiles = ly.Mpad // BM
    sp = -(-2 * n_sms // q_tiles)
    if ws_geo is not None:
        sp = min(sp, -(-ws_geo * S // BQ) * BQ // n_rows_pad)
    sp = min(sp, 2 * math.ceil(math.sqrt(2.0 * n_tiles)))
    sp = max(1, min(sp, n_tiles))
    tps = -(-n_tiles // sp)
    n_splits = -(-n_tiles // tps)
    per_sm = ctas_per_sm(ly.DP)
    grid = q_tiles if n_splits > 1 or MINB > 1 else min(q_tiles, n_sms * per_sm)
    cta_tiles = [range(x, q_tiles, grid) for x in range(grid)]
    return Schedule(B, S, BQ, q_tiles, n_tiles, n_splits, tps, grid, per_sm, cta_tiles)


def batch_for_tiles(N, M, S, T):
    """The smallest batch B with ceil(B S / BQ) == T query tiles whose last tile is partly padded (B S % BQ != 0)."""
    BQ = layout(N, M).BQ
    B = (T - 1) * BQ // S + 1
    while -(-B * S // BQ) == T:
        if B * S % BQ:
            return B
        B += 1
    raise ValueError('no batch of %d tiles with a padded last tile (S = %d, BQ = %d)' % (T, S, BQ))


def tile_geos(sched, t):
    """The geometries with at least one of their S rows in query tile t."""
    return range(t * sched.BQ // sched.S, min(sched.B, ((t + 1) * sched.BQ - 1) // sched.S + 1))


def schedule_rows(sched, ctas):
    """The geometries whose rows lie in the first or the last query tile of each CTA in `ctas`."""
    out = set()
    for x in ctas:
        tiles = sched.cta_tiles[x]
        if len(tiles):
            for t in (tiles[0], tiles[-1]):
                out.update(tile_geos(sched, t))
    return sorted(out)


def ragged_round_rows(sched):
    """The geometries of the last round of query tiles when only some CTAs have a tile in it (else none)."""
    if sched.q_tiles % sched.grid == 0:
        return []
    t0 = sched.q_tiles // sched.grid * sched.grid
    return list(range(tile_geos(sched, t0)[0], sched.B))


def straddling_geos(sched):
    """The geometries whose S rows lie in two query tiles."""
    b = np.arange(sched.B)
    return b[b * sched.S // sched.BQ != ((b + 1) * sched.S - 1) // sched.BQ]


def n_terms(M, S, D):
    """k of the bound: M S (training point, permutation) terms per output plus the descriptor length."""
    return M * S + D


# ------------------------------------------------------------------------------------------------ periodic cells
def _pair_frac(R, lattice_inv):
    """Pair differences d = r_a - r_b (B, D, 3) in tril order and their fractional coordinates lat_inv @ d."""
    R = np.asarray(R, dtype=np.float64)
    r = R.reshape(R.shape[0], -1, 3)
    a, b = np.tril_indices(r.shape[1], -1)
    d = r[:, a, :] - r[:, b, :]
    return d, np.einsum('ij,...j->...i', np.asarray(lattice_inv, dtype=np.float64), d)


def skewed_cell(n_atoms):
    """A triclinic cell (lattice vectors as the COLUMNS, as model['lattice']) whose edges, 1.5 ceil(N^(1/3)) + 0.1 A,
    are just longer than the 1.5 A grid of synth.base_geometry spans: pairs three grid steps apart wrap to images
    1.6 A away, and the skew mixes the axes in lat_inv @ d."""
    e = 1.5 * np.ceil(n_atoms ** (1.0 / 3.0) - 1e-9) + 0.1
    A = np.array([[1.0, 0.18, -0.12], [0.0, 0.98, 0.21], [0.0, 0.0, 0.97]])
    return e * A / np.linalg.norm(A, axis=0)


def pbc_margin(R, lattice, lattice_inv):
    """Per geometry of R (B, 3N): the smallest distance of any pair's fractional difference lat_inv @ d (any of its
    three components) from a half-integer.  Near such a tie the engine (whose cell code contracts to FMAs) and the
    oracle (np.einsum) may round to different images, whose Jacobian rows differ in sign: random periodic queries are
    kept at a margin from ties, and exact ties are tested on their own."""
    assert np.asarray(lattice).shape == (3, 3)
    _, c = _pair_frac(R, lattice_inv)
    return np.min(np.abs(c - np.floor(c) - 0.5), axis=(1, 2))


DESC_C = 64


def desc_pbc_bound(R, lattice, lattice_inv):
    """Componentwise bounds (bx (B, D), bg (B, D)) on |x - x_ref| and on each component of |g - g_ref| for the
    descriptor x = 1/|d'| and Jacobian factor g = d'/|d'|^3 of periodic geometries, d' = d - L round(L^-1 d), away
    from rounding ties (both sides pick the same integer k):
      bx = DESC_C u |w|_2 / |d'|^2,   bg = DESC_C u |w|_2 / |d'|^3,   w = |d| + |L| |k|.
    Derivation (per side, u = 2^-53, gamma_n ~ n u): d = r_a - r_b rounds once (u |d|), L k rounds within gamma_3
    |L||k| (k exact), and the subtraction once more, so |dd'| <= gamma_5 w componentwise -- relative to w, not to |d'|:
    the cancellation in d - L k is what the bound must cover, and |w| / |d'| >= 1 measures it.  Then |d'| moves by at
    most 5u |w| + 2u |d'| (sum of squares and sqrt), x by 9u |w| / |d'|^2 (with the division), and g_c =
    d'_c / |d'|^3 by (|dd'_c| + 3 |d'_c| d|d'| / |d'|) / |d'|^3 + 6u |g_c| <= 26u |w| / |d'|^3.  Two sides: 18u and 52u;
    DESC_C = 64 leaves margin for the FMA-contracted forms."""
    assert np.asarray(lattice).shape == (3, 3)
    L = np.asarray(lattice, dtype=np.float64)
    d, c = _pair_frac(R, lattice_inv)
    k = np.around(c)
    dp = d - np.einsum('ij,...j->...i', L, k)
    w = np.abs(d) + np.einsum('ij,...j->...i', np.abs(L), np.abs(k))
    wn = np.sqrt(np.sum(w * w, axis=-1))
    dist = np.sqrt(np.sum(dp * dp, axis=-1))
    return DESC_C * U * wn / dist ** 2, DESC_C * U * wn / dist ** 3


# ------------------------------------------------------------------------------------------------ magnitude
def _abs_jt(r_d_desc, w):
    """|J|^T w for w >= 0: every pair d = (a, b) adds |g_d| w_d to both atoms (vec_dot_d_desc with all signs +)."""
    D = r_d_desc.shape[0]
    N = int(round((1 + np.sqrt(1 + 8 * D)) / 2))
    a, b = np.tril_indices(N, -1)
    t = np.abs(r_d_desc) * w[:, None]
    out = np.zeros((N, 3))
    np.add.at(out, a, t)
    np.add.at(out, b, t)
    return out.ravel()


def predict_abs_scale(model, R=None, oracle=None, R_desc=None, R_d_desc=None):
    """Per-output magnitudes (scale_E (B,), scale_F (B, 3N)) for `check_predict`.

    The oracle's Predictor._raw with every term replaced by its absolute value, scaled by |std|:
      F_desc: sum_k |c1_k| A_k + |c2_k| |JA_k|,   E: sum_k |a_k| |c2_k|  (+ |alphas_E| terms),
      c1_k = |a_k| base_k 5/sig (+ |alphas_E_k| |c2_k|),  c2_k = base_k (norm_k + sig),  |a_k| = A_k . |JA_k|,
    then F = |J|^T F_desc.  Two refinements make it bound the kernel's arithmetic as well as the oracle's:
      * A_k = |q_k| + |x_k| in place of |diff_k| = |q_k - x_k|, with q, x the query and training descriptors centred
        on the training mean as the engine stores them: the kernel forms sum_k c1 diff_k as (sum_k c1) q - sum_k c1 x_k,
        and a_k as q.JA_k - x_k.JA_k, so its rounding scales with |q| + |x|, not with their difference;
      * the error of the expanded squared distance (see check_predict) through the Matern factors, with
        rho_k = |q_k|^2 + |x_k|^2:  dc1_k = base_k (5/sig) 2 sqrt5 |JA_k|_2 rho_k / sig,  dc2_k = base_k 5 rho_k / sig,
        added to |c1_k| and |c2_k|; with alphas_E also the energy-energy factor's,
        |alphas_E_k| (5/3) (1 + n_k/sig) e_k rho_k / sig^2, added to E.
    model: the model dict; oracle: an oracle.predict.Predictor of it (built if None).  R (B, 3N) queries, or R=None
    with R_desc (B, D) / R_d_desc (B, D, 3) given (the training-point evaluation)."""
    from oracle import desc as odesc
    from oracle import predict as opredict

    op = oracle if oracle is not None else opredict.Predictor(model)
    if R is not None:
        R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * op.n_atoms)
        R_desc, R_d_desc = odesc.from_R(R, op.lat_and_inv)
    R_desc = np.asarray(R_desc, dtype=np.float64)
    R_d_desc = np.asarray(R_d_desc, dtype=np.float64)
    X = np.asarray(model['R_desc'], dtype=np.float64).T  # (M, D)
    M, D = X.shape
    S = op.n_perms
    mu = X.mean(axis=0)
    Xp = op.R_desc_perms  # (M S, D): row m S + p = X_m[tril_perm_p]
    mu_p = np.tile(op._perm_cache(mu[None]), (M, 1))  # (M S, D): row m S + p = mu[tril_perm_p]
    xc = np.abs(Xp - mu_p)
    JAa = np.abs(op.R_d_desc_alpha_perms)
    JA2 = np.sqrt(np.sum(JAa * JAa, axis=1))
    xc2 = np.sum(xc * xc, axis=1)
    ae = np.abs(op.alphas_E_lin) if op.alphas_E_lin is not None else None
    sig = op.sig
    sqrt5 = np.sqrt(5.0)
    B = R_desc.shape[0]
    sE = np.empty(B)
    sF = np.empty((B, 3 * op.n_atoms))
    for i in range(B):
        r = R_desc[i]
        diff = r[None, :] - Xp
        norm = sqrt5 * np.sqrt(np.sum(diff * diff, axis=1))
        e = np.exp(-norm / sig)
        base = e * 5.0 / (3 * sig ** 3)
        qc = np.abs(r[None, :] - mu_p)
        A = qc + xc
        rho = np.sum(qc * qc, axis=1) + xc2
        a_abs = np.einsum('kd,kd->k', A, JAa)
        c2 = base * (norm + sig) + base * 5.0 * rho / sig
        c1 = a_abs * base * 5.0 / sig + base * (5.0 / sig) * 2 * sqrt5 * JA2 * rho / sig
        E = a_abs.dot(c2)
        if ae is not None:
            c1 = c1 + ae * c2
            E += ae.dot((1 + (norm / sig) * (1 + norm / (3 * sig))) * e)
            E += ae.dot((5.0 / 3.0) * (1 + norm / sig) * e * rho / sig ** 2)
        Fd = c1.dot(A) + c2.dot(JAa)
        sE[i] = E
        sF[i] = _abs_jt(R_d_desc[i], Fd)
    std = abs(op.std)
    return sE * std, sF * std


# ------------------------------------------------------------------------------------------------ the check
CHECK_C = 8


def tau(k):
    return CHECK_C * k * U


def check_predict(E, F, E_ref, F_ref, scale, k, what='predict'):
    """|F - F_ref| <= tau scale_F and |E - E_ref| <= tau scale_E + u (|E| + |E_ref|) componentwise, tau = c k u with
    c = CHECK_C = 8 and k = n_terms(M, S, D); plus the global rel_err < 1e-10 of the older tests.  E may be None (a
    return_E=False call).  Returns (max |F - F_ref| / scale_F, max |E - E_ref| / scale_E) for reporting.

    Derivation of c (u = 2^-53, gamma_n = n u / (1 - n u); every error below is relative to the matching term of
    predict_abs_scale, whose terms dominate the absolute values of everything the kernel and the oracle add up):
      * S1 = q.x and S2 = q.JA over the padded descriptor (GEMM1), the row norms |q|^2, |x|^2 and x.JA:
        gamma_D each, so a = S2 - x.JA is within gamma_{D+1} of A.|JA|.
      * exp_neg: Cody-Waite reduction with a two-part ln 2 (exact to ~2^-70 over the range used) and a degree-12 Taylor
        polynomial (truncation 1.7e-16 < 2u for |r| <= ln2/2) evaluated by Estrin in 9 FMAs (<= 5 roundings on the
        longest path, each of a quantity <= 1.5 e^r): e within 10u.  n = x rsqrt(x) adds 2u to n, hence 2u n/sig <= 2u
        of e wherever n <= sig (and base decays faster than any such term grows beyond).  c1 = a (e k_c1) and
        c2 = (e k_base)(n + sig) add 5 roundings (k_base, k_c1 each carry 3): c1, c2 within gamma_{D+1} + 17u.
      * Expanded distance x5 = 5(|q|^2 + |x|^2 - 2 q.x): it differs from 5|diff|^2 by up to
        dx5 <= 5 gamma_{D+2} (|q|^2 + |x|^2 + 2|q.x|) <= 10 gamma_{D+2} rho.  Matern-5/2 is flat at n = 0:
        d/dn [(n + sig) e^{-n/sig}] = -(n/sig) e^{-n/sig}, so c2 moves by k_base e (n/sig) dn <= k_base e dx5 / (2 sig)
        (dn <= dx5 / (2n)): second order in n, the dc2 term of predict_abs_scale times 10 gamma_{D+2} / 10.  c1 moves to
        first order through e' = -e/sig: by a k_c1 e dn / sig with |a| <= (n/sqrt5)|JA|_2, i.e. at most
        k_c1 e |JA|_2 dx5 / (2 sqrt5 sig) -- the dc1 term times gamma_{D+2} (2 sqrt5 absorbs 10 / (2 sqrt5) = sqrt5).
        As n -> 0 (a query on a training point) a itself is rounding noise and the same bound holds with dn <= sqrt(dx5).
        With alphas_E, K_ee = (1 + (n/sig)(1 + n/(3 sig))) e^{-n/sig} is flat at n = 0 too: dK_ee/dn =
        -(n/(3 sig^2))(1 + n/sig) e^{-n/sig}, so with dn <= dx5/(2n) and dx5 <= 10 gamma_{D+2} rho it moves by at most
        gamma_{D+2} (5/3)(1 + n/sig) e rho / sig^2 -- the K_ee term of predict_abs_scale times gamma_{D+2}.
      * GEMM2 and the row sums: G = (sum_m c1) q - sum_m (c1 x + c2 JA), 2M + 1 terms per virtual row: gamma_{2M+1}.
        The finishing kernel adds the S permutations times the split count (<= 2 sqrt(2 Mpad/BM) + 1), J^T adds
        N - 1 terms per force component, std one rounding: together gamma_{S(sp+1) + N + 1}.
    The kernel's error is therefore within gamma_{2M + D + S(sp+1) + N + 25} of the scale, and the FP64 oracle's (direct
    differences, sums over the M S cache rows and N atoms) within gamma_{MS + D + N + 10}.  For every shape with
    S >= 2 or M >= D + N + 40 (all the tests use), both totals are below 3 k u, so |F - F_ref| <= 6 k u (1 + O(ku)) scale;
    c = 8 leaves margin for the x5 terms folded in above.  E sums the same a c2 terms and carries the integration
    constant c, which is not part of any sum: adding it rounds once per side, hence the u (|E| + |E_ref|).
    A NaN anywhere fails the check (NaN <= bound is false)."""
    sE, sF = scale
    t = tau(k)
    F = np.asarray(F, dtype=np.float64)
    F_ref = np.asarray(F_ref, dtype=np.float64)
    errF = np.abs(F - F_ref)
    okF = errF <= t * sF
    if not np.all(okF):
        bad = np.argwhere(~okF)
        i = tuple(int(j) for j in bad[0])
        raise AssertionError(
            '%s: %d force entries outside tau = %.2e times the scale; first at %s: |err| %r > %r (|err|/scale %.2e)'
            % (what, bad.shape[0], t, i, float(errF[i]), float(t * sF[i]), float(errF[i] / sF[i]))
        )
    ratio_E = None
    if E is not None:
        E = np.asarray(E, dtype=np.float64)
        E_ref = np.asarray(E_ref, dtype=np.float64)
        errE = np.abs(E - E_ref)
        okE = errE <= t * sE + U * (np.abs(E) + np.abs(E_ref))
        if not np.all(okE):
            i = int(np.argwhere(~okE)[0][0])
            raise AssertionError('%s: %d energies outside the bound; first at %d: |err| %r > %r'
                                 % (what, int(np.sum(~okE)), i, float(errE[i]), float(t * sE[i])))
        ratio_E = float(np.max(errE / sE))
        relE = float(np.max(errE) / max(np.max(np.abs(E_ref)), 1e-300))
        if not relE < 1e-10:
            raise AssertionError('%s: energy rel_err %.3e >= 1e-10' % (what, relE))
    relF = float(np.max(errF) / max(np.max(np.abs(F_ref)), 1e-300))
    if not relF < 1e-10:
        raise AssertionError('%s: force rel_err %.3e >= 1e-10' % (what, relF))
    return float(np.max(errF / sF)), ratio_E
