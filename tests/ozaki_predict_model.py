"""Stage-by-stage model of the large-descriptor predictor (D > 256: `run_queries` in csrc/predict.cu) in NumPy, with the
checks that hold each stage to it, and a composed error bound of the int8-slice form against the FP64 oracle.

The GEMM-composed predictor runs, per chunk of rows = n_geo * n_perms virtual query rows:
  Qg, qq       query rows x[pinv_p] - mu (zero beyond D) and their squared norms
  S1, S2       Qg Xc^T and Qg JA^T                                      (GEMM, k = DS; overwrite)
  C1, C2       k_transform_rows in place: the Matern factors, csum = sum_m C1, Erow = the energy terms
  acc          C1 XcT^T, then + C2 JAT^T                                 (GEMM, k = Mpad; overwrite, then accumulate)
  G            k_combine_rows: csum Qg - acc
  E, F         fold of the n_perms rows of a query through perm_p, F = std J^T F_desc, E = std sum Erow + c
With oz_s >= 2 the four GEMMs run on the int8-slice GEMM, which tests/ozaki_model.py states bit for bit, so the checks
compare every contraction bit for bit with `om.gemm` on the operands the kernel was fed.  The FP64 stages between them
get componentwise FP64 tolerances (derived in `check_transform`, `check_combine`, `check_finish`), and `e2e_bound`
bounds E and F of the whole int8 composition against the oracle.

`stages(...)` is the NumPy stand-in for the device's taps (sgdml_b200_predict_stages): a dict with the same keys, so
the same checks run on both; its `defect` argument injects the faults the checks must reject (`DEFECTS`)."""

import numpy as np

import ozaki_model as om
import predict_checks as pc

U = 2.0 ** -53
SQRT5 = np.sqrt(5.0)
DEFECTS = ('gemm1_short', 'gemm2_short', 'gemm3_short', 'gemm4_short', 'stale_ja', 'foreign_xc', 'c1_exponent',
           'gemm4_overwrite', 'drop_pair', 'drop_ae', 'stale_row', 'c1_padding')


# ------------------------------------------------------------------------------------------------ model layout
def layout_arrays(model, alphas_E=None):
    """The engine's padded model matrices (sgdml_b200_model_create / set_alphas): a dict with X (M, D), mu (DS), Xc, JA
    (Mpad, DS), XcT, JAT (DP, Mpad), mm, xja, ae (Mpad), perm, pinv (n_perms, D), M, D, DP, DS, Mpad, sig, std, c."""
    X = np.ascontiguousarray(np.asarray(model['R_desc'], dtype=np.float64).T)
    M, D = X.shape
    N = int(np.asarray(model['z']).shape[0])
    ly = pc.layout(N, M)
    assert ly.large, 'the GEMM-composed predictor runs for D > 256 only'
    DP, Mpad = ly.DP, ly.Mpad
    DS = DP + 4
    mu = np.zeros(DS)
    mu[:D] = X.mean(axis=0)
    Xc = np.zeros((Mpad, DS))
    Xc[:M, :D] = X - mu[:D]
    JA = np.zeros((Mpad, DS))
    JA[:M, :D] = np.asarray(model['R_d_desc_alpha'], dtype=np.float64)
    ae = np.zeros(Mpad)
    if alphas_E is None and 'alphas_E' in model:
        alphas_E = model['alphas_E']
    if alphas_E is not None:
        ae[:M] = np.asarray(alphas_E, dtype=np.float64)
    lin = np.asarray(model['tril_perms_lin'], dtype=np.int64)
    S = lin.size // D
    perm = (lin.reshape(D, S).T - np.arange(S)[:, None] * D).astype(np.int64)
    pinv = np.empty_like(perm)
    for p in range(S):
        pinv[p, perm[p]] = np.arange(D)
    return dict(X=X, mu=mu, Xc=Xc, JA=JA, XcT=np.ascontiguousarray(Xc[:, :DP].T), JAT=np.ascontiguousarray(JA[:, :DP].T),
                mm=np.sum(Xc * Xc, axis=1), xja=np.sum(Xc * JA, axis=1), ae=ae, use_ae=alphas_E is not None,
                perm=perm, pinv=pinv, M=M, D=D, DP=DP, DS=DS, Mpad=Mpad, N=N, n_perms=S, sig=float(model['sig']),
                std=float(model.get('std', 1.0)), c=float(model['c']))


def query_rows(xq, pinv, mu, DS):
    """Qg (B S, DS) and qq as k_query_rows forms them: row b S + p = x_b[pinv_p] - mu, zero beyond D."""
    xq = np.atleast_2d(np.asarray(xq, dtype=np.float64))
    B, D = xq.shape
    S = pinv.shape[0]
    Qg = np.zeros((B * S, DS))
    for p in range(S):
        Qg[p::S, :D] = xq[:, pinv[p]] - mu[:D]
    return Qg, np.sum(Qg * Qg, axis=1)


# ------------------------------------------------------------------------------------------------ the stages
def _kconst(sig):
    k_base = 5.0 / (3.0 * sig ** 3)
    return k_base, k_base * 5.0 / sig


def transform(S1, S2, qq, mm, xja, ae, M, sig, use_ae):
    """k_transform_rows restated (np.exp for exp_neg): (C1, C2, csum, Erow); C1 = C2 = 0 in the padding columns."""
    k_base, k_c1 = _kconst(sig)
    x5 = np.maximum(5.0 * qq[:, None] + 5.0 * mm[None, :M] - 10.0 * S1[:, :M], 1e-300)
    n = np.sqrt(x5)
    e = np.exp(-n / sig)
    a = S2[:, :M] - xja[None, :M]
    c2 = (e * k_base) * (n + sig)
    c1 = a * (e * k_c1)
    Eterm = a * c2
    if use_ae:
        t = n / sig
        c1 = c1 + ae[None, :M] * c2
        Eterm = Eterm + ae[None, :M] * (1.0 + t * (1.0 + t / 3.0)) * e
    C1 = np.zeros_like(S1)
    C2 = np.zeros_like(S2)
    C1[:, :M] = c1
    C2[:, :M] = c2
    return C1, C2, c1.sum(axis=1), Eterm.sum(axis=1)


def finish(G, Erow, perm, gq, std, c):
    """The finishing kernels: F_desc[d] = sum_p G[b S + p][perm_p[d]], F = std J^T F_desc, E = std sum_p Erow + c."""
    from oracle import desc as odesc

    S, D = perm.shape
    B = G.shape[0] // S
    Fd = np.zeros((B, D))
    for p in range(S):
        Fd += G[p::S][:, perm[p]]
    F = odesc.vec_dot_d_desc(gq, Fd) * std
    E = Erow.reshape(B, S).sum(axis=1) * std + c
    return E, F, Fd


def _gemm(A, B, S, C0=None, product=None, defect=None):
    """One contraction as the engine runs it: FP64 (S = 0; here a NumPy matmul) or the int8-slice GEMM `om.gemm`."""
    C = np.zeros((A.shape[0], B.shape[0])) if C0 is None else C0
    if S == 0:
        return C + A @ B.T if C0 is not None else A @ B.T
    lev = None if defect is not None or product is None else om.operands(A, B, S, product)
    return om.gemm(A, B, C, 1.0, S, overwrite=C0 is None, defect=defect, lev=lev)


def stages(arr, Qg, qq, S, defect=None, prev=None, product=None):
    """The taps of one chunk as the engine with `S` slices (0: FP64) produces them, from the model arrays `arr` and
    the query rows.  defect (one of DEFECTS) injects a fault; 'stale_ja' needs prev = the arrays before set_alphas,
    'foreign_xc' prev = another model's arrays, 'stale_row' prev = the previous chunk's Qg."""
    M, Mpad = arr['M'], arr['Mpad']
    Xc, JA, XcT, JAT = arr['Xc'], arr['JA'], arr['XcT'], arr['JAT']
    Qin = Qg
    if defect == 'stale_row':
        Qin, qq = Qg.copy(), qq.copy()
        Qin[0] = prev[-1]
        qq[0] = np.sum(prev[-1] * prev[-1])
    if defect == 'stale_ja':
        JA, JAT = prev['JA'], prev['JAT']
    if defect == 'foreign_xc':
        Xc = prev['Xc']
    s1 = S - 1 if defect == 'gemm1_short' else S
    s2 = S - 1 if defect == 'gemm2_short' else S
    S1 = _gemm(Qin, Xc, s1, product=product)
    S2 = _gemm(Qin, JA, s2, product=product)
    ae = arr['ae'].copy()
    if defect == 'drop_ae':
        ae[M // 2] = 0.0
    C1, C2, csum, Erow = transform(S1, S2, qq, arr['mm'], arr['xja'], ae, M, arr['sig'], arr['use_ae'])
    C1in = C1
    if defect == 'c1_padding':
        assert Mpad > M, 'the defect needs padding columns'
        C1in = C1.copy()
        C1in[:, M] = C1[:, 0]
    s3 = S - 1 if defect == 'gemm3_short' else S
    s4 = S - 1 if defect == 'gemm4_short' else S
    acc = _gemm(C1in, XcT, s3, product=product, defect='row_exponent' if defect == 'c1_exponent' else None)
    if defect == 'gemm4_overwrite':
        acc = _gemm(C2, JAT, s4, product=product)
    else:
        acc = _gemm(C2, JAT, s4, C0=acc, product=product, defect='drop_pair' if defect == 'drop_pair' else None)
    G = csum[:, None] * Qin[:, :arr['DP']] - acc
    return dict(Qg=Qin, qq=qq, S1=S1, S2=S2, C1=C1in, C2=C2, csum=csum, Erow=Erow, acc=acc, G=G, oz_s=S)


# ------------------------------------------------------------------------------------------------ the checks
def _fail(what, bad, got, want, tol=None):
    i = tuple(int(j) for j in np.argwhere(bad)[0])
    msg = '%s: %d entries wrong; first at %s: %r vs %r' % (what, int(np.sum(bad)), i, float(got[i]), float(want[i]))
    if tol is not None:
        msg += ' (tolerance %.3g)' % float(tol[i])
    raise AssertionError(msg)


def check_exact(what, got, want):
    """Bit-identical (NaN in the same places)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, '%s: shape %s vs %s' % (what, got.shape, want.shape)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if np.any(bad):
        _fail(what, bad, got, want)


def check_within(what, got, want, tol):
    err = np.abs(np.asarray(got) - np.asarray(want))
    bad = ~(err <= tol)
    if np.any(bad):
        _fail(what, bad, np.asarray(got), np.asarray(want), np.broadcast_to(tol, err.shape))


def check_query_rows(t, arr, xq):
    """Qg bit-identical to x[pinv_p] - mu (one subtraction per entry; xq: the descriptors the kernel read, e.g. the
    training descriptors for R = NULL), qq within 1.01 DS u qq (the kernel's fma chain and shuffle tree sum in another
    order)."""
    Qg, qq = query_rows(xq, arr['pinv'], arr['mu'], arr['DS'])
    check_exact('Qg (query rows)', t['Qg'], Qg)
    check_within('qq (query rows)', t['qq'], qq, 1.01 * arr['DS'] * U * qq)


def check_contractions(t, arr, S, product=None):
    """The four contractions bit for bit against `om.gemm` (S >= 2) on the operands the taps show: S1, S2 from Qg, the
    accumulator from C1, C2.  For S = 0 the FP64 GEMM is held to gamma_k of |A| |B|^T instead (its own bit-level
    tests are tests/test_gemm_classes.py).  Raises AssertionError naming the contraction."""
    Qg, C1, C2 = t['Qg'], t['C1'], t['C2']
    pairs = (('S1 = Qg Xc^T', t['S1'], Qg, arr['Xc'], None), ('S2 = Qg JA^T', t['S2'], Qg, arr['JA'], None))
    if S == 0:
        for what, got, A, B, _ in pairs:
            check_within(what, got, A @ B.T, 1.01 * A.shape[1] * U * (np.abs(A) @ np.abs(B).T))
        want = C1 @ arr['XcT'].T + C2 @ arr['JAT'].T
        k = 2 * C1.shape[1]
        tol = 1.01 * k * U * (np.abs(C1) @ np.abs(arr['XcT']).T + np.abs(C2) @ np.abs(arr['JAT']).T)
        check_within('acc = C1 XcT^T + C2 JAT^T', t['acc'], want, tol)
        return
    for what, got, A, B, _ in pairs:
        check_exact(what + ' (%d slices)' % S, got, _gemm(A, B, S, product=product))
    first = _gemm(C1, arr['XcT'], S, product=product)
    check_exact('acc = C1 XcT^T + C2 JAT^T (%d slices)' % S, t['acc'], _gemm(C2, arr['JAT'], S, C0=first,
                                                                               product=product))


def transform_tol(t, arr):
    """Componentwise tolerances (tol_C1, tol_C2, tol_csum, tol_Erow) of k_transform_rows against `transform` on the same
    S1, S2 (u = 2^-53):
      * a = S2 - xja is one subtraction on both sides: bit-identical.
      * x5 = fma(-10, s1, 5 qq + 5 mm) against 5 qq + 5 mm - 10 s1: the kernel rounds twice (5 mm, then the sum inside
        the fma), the model four times; so the two differ by dx5 <= 6 u (|5 qq| + |5 mm| + |10 s1|) -- relative to
        those magnitudes, not to x5: at a training point they cancel to rounding noise.
      * n = sqrt(x5) moves by dn <= min(dx5 / n, sqrt(dx5)) (n dn <= d(n^2); the sqrt form as n -> 0), plus 2u n
        (x rsqrt(x) against sqrt).  exp_neg is within 10u of exp (its docstring in predict_checks.check_predict),
        e^(-n/sig) moves by e dn / sig.
      * c2 = (e k_base)(n + sig): Matern-5/2 is flat at n = 0 (d c2/dn = -k_base (n/sig) e), so dn enters as
        k_base e dn n / sig <= k_base e dx5 / sig; plus 16u |c2| for the roundings (k_base carries 3, e 10, 3 more).
      * c1 = a (e k_c1) (+ ae c2): |a| e k_c1 dn / sig, plus 20u |c1|, plus |ae| times c2's tolerance.
      * K_ee = (1 + t(1 + t/3)) e, t = n/sig: dK_ee/dn = -(t/(3 sig))(1 + t) e, so |ae| dn (1 + t) e t / (3 sig) +
        16u |K_ee|.
      * csum and Erow are sums over M terms in different orders: the sum of the entries' tolerances plus
        1.01 M u sum |terms|."""
    M, sig = arr['M'], arr['sig']
    k_base, k_c1 = _kconst(sig)
    qq, S1, S2 = t['qq'], t['S1'][:, :M], t['S2'][:, :M]
    mm, ae = arr['mm'][:M], arr['ae'][:M] if arr['use_ae'] else np.zeros(M)
    mag = 5.0 * qq[:, None] + 5.0 * mm[None, :] + 10.0 * np.abs(S1)
    x5 = np.maximum(5.0 * qq[:, None] + 5.0 * mm[None, :] - 10.0 * S1, 0.0)
    dx5 = 6 * U * mag
    n = np.sqrt(x5)
    with np.errstate(divide='ignore', invalid='ignore'):
        dn = np.minimum(np.where(n > 0, dx5 / n, np.inf), np.sqrt(dx5)) + 2 * U * n
    n_lo = np.sqrt(np.maximum(x5 - dx5, 0.0))
    e = np.exp(-n_lo / sig) * (1 + 20 * U)
    a = S2 - arr['xja'][None, :M]
    c2 = (e * k_base) * (n + sig)
    tc2 = k_base * e * np.minimum(dx5 / sig, dn * (n + dn) / sig) + 16 * U * c2
    c1 = np.abs(a) * e * k_c1 + np.abs(ae) * c2
    tc1 = np.abs(a) * e * k_c1 * dn / sig + 20 * U * c1 + np.abs(ae) * tc2
    t_ = (n + dn) / sig
    kee = (1 + t_ * (1 + t_ / 3)) * e
    tE = np.abs(a) * tc2 + 2 * U * np.abs(a) * c2 + np.abs(ae) * (dn * (1 + t_) * e * t_ / (3 * sig) + 16 * U * kee)
    Eterm = np.abs(a) * c2 + np.abs(ae) * kee
    tol_csum = tc1.sum(axis=1) + 1.01 * M * U * c1.sum(axis=1)
    tol_E = tE.sum(axis=1) + 1.01 * M * U * Eterm.sum(axis=1)
    pad = np.zeros((S1.shape[0], arr['Mpad'] - M))
    return np.hstack([tc1, pad]), np.hstack([tc2, pad]), tol_csum, tol_E


def check_transform(t, arr):
    """k_transform_rows (C1, C2, csum, Erow) against `transform` on the tapped S1, S2 within `transform_tol`; the
    padding columns m >= M of C1 and C2 must be exactly zero (the accumulator's GEMM contracts over them)."""
    M = arr['M']
    ae = arr['ae']
    C1, C2, csum, Erow = transform(t['S1'], t['S2'], t['qq'], arr['mm'], arr['xja'], ae, M, arr['sig'], arr['use_ae'])
    tc1, tc2, tcs, tE = transform_tol(t, arr)
    check_exact('C1 padding columns (m >= M)', t['C1'][:, M:], np.zeros_like(t['C1'][:, M:]))
    check_exact('C2 padding columns (m >= M)', t['C2'][:, M:], np.zeros_like(t['C2'][:, M:]))
    check_within('C1 (transform)', t['C1'], C1, tc1)
    check_within('C2 (transform)', t['C2'], C2, tc2)
    check_within('csum (transform)', t['csum'], csum, tcs)
    check_within('Erow (transform)', t['Erow'], Erow, tE)


def check_combine(t, arr):
    """G = csum Qg - acc (k_combine_rows; the kernel may contract it to an fma): within 2u (|csum Qg| + |acc|)."""
    Q = t['Qg'][:, :arr['DP']]
    prod = t['csum'][:, None] * Q
    check_within('G (combine)', t['G'], prod - t['acc'], 2 * U * (np.abs(prod) + np.abs(t['acc'])))


def check_finish(t, arr, gq, E, F, scaled=True):
    """E and F from the tapped G and Erow (perm fold, J^T, std, c): each output is a sum of S (fold) and N - 1 (J^T)
    terms, and std rounds once: within gamma_{S + N + 1} of the same sum over absolute values, and E also within
    u |E| for adding c."""
    std, c = (arr['std'], arr['c']) if scaled else (1.0, 0.0)
    E_want, F_want, _ = finish(t['G'], t['Erow'], arr['perm'], gq, std, c)
    _, F_abs = _abs_finish(np.abs(t['G']), arr['perm'], gq, abs(std))
    k = arr['n_perms'] + arr['N'] + 2
    check_within('F (finish)', F, F_want, 1.01 * k * U * F_abs)
    E_abs = np.abs(t['Erow']).reshape(-1, arr['n_perms']).sum(axis=1) * abs(std)
    if E is not None:
        check_within('E (finish)', E, E_want, 1.01 * k * U * E_abs + 2 * U * np.abs(E_want))


def _abs_finish(Gabs, perm, gq, std):
    S, D = perm.shape
    B = Gabs.shape[0] // S
    Fd = np.zeros((B, D))
    for p in range(S):
        Fd += Gabs[p::S][:, perm[p]]
    return Fd, np.stack([pc._abs_jt(gq[b], Fd[b]) for b in range(B)]) * std


def check_stages(t, arr, S, gq=None, E=None, F=None, scaled=True, product=None):
    """Every stage of one tapped chunk: the contractions (bit for bit for S >= 2), the transform, the combine, and
    with gq the finishing of E and F."""
    check_contractions(t, arr, S, product=product)
    check_transform(t, arr)
    check_combine(t, arr)
    if gq is not None:
        check_finish(t, arr, gq, E, F, scaled)


# ------------------------------------------------------------------------------------------------ end to end
def e2e_bound(arr, Qg, qq, gq, S, scale, k_terms, scaled=True):
    """Componentwise bound (bE (B,), bF (B, 3N)) on |E - E_oracle| and |F - F_oracle| of the int8-slice composition
    with S slices.  It is the FP64 bound of predict_checks.check_predict (tau scale: the kernel's FP64 arithmetic and
    the oracle's) plus how far the four int8 GEMMs move the exact result, pushed through the stages:

      * GEMM 1, 2 (k = DS): |dS1| <= b1 = method_bound(e_Q, e_Xc), |dS2| <= b2 = method_bound(e_Q, e_JA) per entry
        (tests/ozaki_model.py; the row exponents of Qg, Xc, JA are those the kernel uses).
      * transform: x5 = 5 qq + 5 mm - 10 S1 moves by dx5 = 10 b1, a = S2 - xja by b2.  n = sqrt(x5) moves by
        dn <= min(dx5 / n, sqrt(dx5)) (n dn <= d(n^2)); e = exp(-n/sig) is at most e_hi = exp(-n_lo/sig) on the
        interval, n_lo = sqrt(max(x5 - dx5, 0)).  Matern-5/2 is flat at n = 0: dc2/dx5 = -k_base e / (2 sig), so
        |dc2| <= k_base e_hi dx5 / (2 sig), first order even at a training point's self-pair (n = 0).  c1 = a e k_c1:
        |dc1| <= k_c1 (b2 e_hi + |a| e_hi dn / sig) with |a| <= n |JA|_2 / sqrt5 (Cauchy-Schwarz: a = delta . JA, n =
        sqrt5 |delta|), so |a| dn <= |JA|_2 dx5 / sqrt5 also at n = 0; |a| is taken as the smaller of that and the
        FP64 |a| plus gamma_DS (|Qg| + |Xc|) . |JA|.  With alphas_E: + |ae| |dc2| in c1, and K_ee moves by at most
        dx5 / (6 sig^2) ((1 + t) e^-t <= 1).  csum and Erow add these over m.
      * GEMM 3, 4 (k = Mpad): acc moves by |dC1| |XcT|^T + |dC2| |JAT|^T plus method_bound(e_C1, e_XcT) +
        method_bound(e_C2, e_JAT), with e_C the row exponents of |C| + |dC| (the computed C1 may sit one exponent
        higher at a power-of-two boundary: this covers it).
      * combine: dG = |dcsum| |Qg| + |dacc|; the fold over permutations adds the S rows of a query, F = std |J|^T dF_desc,
        E = std sum_p dErow.
    The magnitudes (S1, S2, C1, C2, x5) are those of the FP64 chain on the same Qg; their own rounding is within the
    tau term.  Returns (bE, bF, parts) with parts the int8 terms alone (zero for S = 0)."""
    M, DS, Mpad, sig = arr['M'], arr['DS'], arr['Mpad'], arr['sig']
    std = abs(arr['std']) if scaled else 1.0
    k_base, k_c1 = _kconst(sig)
    sE, sF = scale
    t = pc.tau(k_terms)
    B = Qg.shape[0] // arr['n_perms']
    if S == 0:
        z = (np.zeros(B), np.zeros(sF.shape))
        return t * sE, t * sF, z
    Xc, JA = arr['Xc'], arr['JA']
    eq, _ = om.row_exponents(Qg)
    ex, _ = om.row_exponents(Xc)
    ej, _ = om.row_exponents(JA)
    b1 = om.method_bound(eq, ex, DS, S)[:, :M]
    b2 = om.method_bound(eq, ej, DS, S)[:, :M]
    S1 = (Qg @ Xc.T)[:, :M]
    S2 = (Qg @ JA.T)[:, :M]
    x5 = np.maximum(5.0 * qq[:, None] + 5.0 * arr['mm'][None, :M] - 10.0 * S1, 0.0)
    dx5 = 10.0 * b1
    n = np.sqrt(x5)
    with np.errstate(divide='ignore', invalid='ignore'):
        dn = np.minimum(np.where(n > 0, dx5 / n, np.inf), np.sqrt(dx5))
    n_lo = np.sqrt(np.maximum(x5 - dx5, 0.0))
    e_hi = np.exp(-n_lo / sig)
    a_fp = np.abs(S2 - arr['xja'][None, :M]) + 1.01 * DS * U * (np.abs(Qg) @ np.abs(JA).T
                                                                  + np.sum(np.abs(Xc * JA), axis=1)[None, :])[:, :M]
    ja2 = np.sqrt(np.sum(JA * JA, axis=1))[None, :M]
    a_dn = np.minimum(a_fp * dn, ja2 * dx5 / SQRT5)
    dc2 = k_base * e_hi * dx5 / (2 * sig)
    ae = np.abs(arr['ae'][None, :M]) if arr['use_ae'] else np.zeros((1, M))
    dc1 = k_c1 * (b2 * e_hi + e_hi * a_dn / sig) + ae * dc2
    c2_hi = k_base * e_hi * (n_lo + sig)
    dE_row = np.sum(b2 * c2_hi + (a_fp + b2) * dc2 + ae * dx5 / (6 * sig ** 2), axis=1)
    dcsum = dc1.sum(axis=1)
    C1, C2, _, _ = transform(Qg @ Xc.T, Qg @ JA.T, qq, arr['mm'], arr['xja'], arr['ae'], M, sig, arr['use_ae'])
    pad = np.zeros((Qg.shape[0], Mpad - M))
    dC1, dC2 = np.hstack([dc1, pad]), np.hstack([dc2, pad])
    e1, _ = om.row_exponents(np.abs(C1) + dC1)
    e2, _ = om.row_exponents(np.abs(C2) + dC2)
    XcT, JAT = arr['XcT'], arr['JAT']
    ext, _ = om.row_exponents(XcT)
    ejt, _ = om.row_exponents(JAT)
    dacc = (dC1 @ np.abs(XcT).T + dC2 @ np.abs(JAT).T + om.method_bound(e1, ext, Mpad, S)
            + om.method_bound(e2, ejt, Mpad, S))
    dG = dcsum[:, None] * np.abs(Qg[:, :arr['DP']]) + dacc
    _, dF = _abs_finish(dG, arr['perm'], gq, std)
    dE = dE_row.reshape(B, arr['n_perms']).sum(axis=1) * std
    return t * sE + dE * (1 + 1e-6), t * sF + dF * (1 + 1e-6), (dE, dF)


def check_e2e(E, F, E_ref, F_ref, bound, what):
    """|E - E_ref| <= bE + u (|E| + |E_ref|) (c rounds once per side) and |F - F_ref| <= bF componentwise.  Returns the
    worst ratios (max |dF| / bF, max |dE| / bE)."""
    bE, bF = bound[0], bound[1]
    errF = np.abs(np.asarray(F) - F_ref)
    check_within(what + ': F against the oracle', F, F_ref, bF)
    rF = float(np.max(errF / bF))
    rE = None
    if E is not None:
        errE = np.abs(np.asarray(E) - E_ref)
        check_within(what + ': E against the oracle', E, E_ref, bE + U * (np.abs(E) + np.abs(E_ref)))
        rE = float(np.max(errE / bE))
    return rF, rE


# ------------------------------------------------------------------------------------------------ fixtures
KINDS = ('plain', 'ecstr', 'pbc', 'perms')


def make_model(N, M, kind, seed=0, sig=30.0, perms=None, r0=None):
    """A random-coefficient model of one kind and its training data: (model, R (M, 3N), R_d_desc (M, D, 3)).
      plain  the identity permutation only
      ecstr  two permutations and seeded mixed-sign alphas_E that move E and F by well over 10 %
      pbc    two permutations, training descriptors in the skewed cell of predict_checks.skewed_cell
      perms  the rotor-and-swap group of synth (6 permutations), or `perms` when given
    std and c are away from 1 and 0, so the finishing is tested too."""
    from oracle import desc as odesc
    from sgdml_b200 import synth

    if kind == 'plain':
        P = np.arange(N)[None]
    elif kind == 'perms':
        P = synth.rotor_swap_group(N, 1, 1) if perms is None else np.asarray(perms)
    else:
        P = synth.rotor_swap_group(N, 0, 1)
    R = synth.geometries(N, M, seed, r0=r0).reshape(M, -1)
    lat = pc.skewed_cell(N) if kind == 'pbc' else None
    lat_and_inv = None if lat is None else (lat, np.linalg.inv(lat))
    x, g = odesc.from_R(R, lat_and_inv)
    rng = np.random.default_rng(seed + 99)
    alphas = rng.standard_normal(M * 3 * N)
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
        'perms': np.asarray(P, dtype=np.int64),
        'tril_perms_lin': odesc.tril_perms_lin(np.asarray(P, dtype=np.int64)),
        'use_E': True,
    }
    if kind == 'ecstr':
        model['alphas_E'] = 3.0 * rng.standard_normal(M)
    if lat is not None:
        model['lattice'] = lat
    return model, R, g


def queries(model, B, seed):
    """B seeded query geometries near the training set; in a periodic model's cell, away from rounding ties."""
    from sgdml_b200 import synth

    N = int(np.asarray(model['z']).shape[0])
    if 'lattice' not in model:
        return synth.geometries(N, B, seed).reshape(B, -1)
    lat = np.asarray(model['lattice'])
    R = synth.geometries(N, 2 * B, seed).reshape(2 * B, -1)
    keep = pc.pbc_margin(R, lat, np.linalg.inv(lat)) >= 1e-6
    return np.ascontiguousarray(R[keep][:B])


def oracle_case(model, R=None, train=None):
    """(E_ref, F_ref, x (B, D), g (B, D, 3), scale, k) from the oracle: R queries, or train = (R_desc, R_d_desc) rows
    of training points (scaled outputs)."""
    from oracle import desc as odesc
    from oracle import predict as opredict

    op = opredict.Predictor(model)
    if R is not None:
        x, g = odesc.from_R(R, op.lat_and_inv)
        E, F = op.predict(R)
    else:
        x, g = train
        op.set_R_desc(x)
        op.set_R_d_desc(g)
        E, F = op.predict(None)
    scale = pc.predict_abs_scale(model, oracle=op, R_desc=x, R_d_desc=g)
    M, D = np.asarray(model['R_desc']).T.shape
    return E, F, x, g, scale, pc.n_terms(M, op.n_perms, D)
