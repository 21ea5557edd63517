"""Exact model of the int8-slice GEMM k_ozaki_gemm<S> (csrc/ozaki.cu), bit for bit, in NumPy.

The kernel's arithmetic is fully determined, so the model restates it operation by operation:

  row exponent  e = 0 for a zero row, otherwise frexp(max |x|)[1] + 1, so that |x| 2^-e < 1/2
  slices        v = ldexp(x, -e); S times: v *= 2^7, q_p = rint(v) (half to even, as CUDA's rint), v -= q_p
  levels        Lev_L = sum_{p + q = L, p, q <= S} A_p B_q^T for L = 2 .. S + 1 (pairs with p + q > S + 1 are dropped).
                Every partial sum is an integer below 2^31, so a float64 matmul of the integer-valued slices, in any
                summation order, is exact.
  sum           V = 0; for L = S + 1 down to 2: V = V + Lev_L 2^(-7 L)  (the kernel's fma: the product is exact)
  update        U = ldexp(fl(alpha V), e_A,i + e_B,j);  C = fl(C0 + U), or C = U when overwriting
  non-finite    every entry of C whose row of A or row of B holds a NaN or an infinity is NaN
  tri           the kernel updates every entry of each 128 x 32 tile (tm, tn) with 32 tn <= 128 tm + 127, entries
                above the diagonal included; every other entry keeps its bits

`method_bound` is the componentwise error of U against alpha (A B^T) computed exactly; its derivation is in its
docstring.  `gemm(..., defect=...)` injects the synthetic defects the exact comparison must reject."""

import numpy as np

BITS = 7
BM, BN = 128, 32  # the kernel's tile of C
K_MAX = 1 << 14  # int32 headroom: 64^2 k S < 2^31
U64 = 2.0 ** -53
DEFECTS = ('drop_pair', 'level_weight', 'row_exponent', 'tile_twice', 'b_tile_rows', 'ignore_overwrite')


def row_exponents(X):
    """(e, bad): the kernel's row exponents, and which rows hold a NaN or an infinity (their e is reported as 0 here;
    the kernel marks them with a sentinel and slices them as zero rows)."""
    X = np.asarray(X, dtype=np.float64)
    bad = ~np.all(np.isfinite(X), axis=1)
    amax = np.max(np.abs(np.where(bad[:, None], 0.0, X)), axis=1, initial=0.0)
    e = np.zeros(X.shape[0], dtype=np.int64)
    nz = amax > 0
    e[nz] = np.frexp(amax[nz])[1] + 1
    return e, bad


def split(X, S, e_shift=None):
    """(e, slices, bad): slices is (S, rows, k) float64 holding the integers q_p, |q_p| <= 64.  e_shift: per-row
    exponent offsets (a defect)."""
    X = np.asarray(X, dtype=np.float64)
    e, bad = row_exponents(X)
    if e_shift is not None:
        e = e + e_shift
    v = np.ldexp(np.where(bad[:, None], 0.0, X), -e[:, None])
    out = np.empty((S,) + X.shape)
    for p in range(S):
        v = v * float(1 << BITS)
        q = np.rint(v)
        out[p] = q
        v = v - q
    return e, out, bad


def level_pairs(S, L):
    """The slice pairs (p, q) of level L = p + q that the kernel multiplies."""
    return [(p, L - p) for p in range(max(1, L - S), min(S, L - 1) + 1)]


def levels(sa, sb, S, drop=()):
    """[Lev_2, ..., Lev_{S+1}] as exact float64 integers; drop: pairs (p, q) left out (a defect)."""
    out = []
    for L in range(2, S + 2):
        pairs = [pq for pq in level_pairs(S, L) if pq not in drop]
        if not pairs:
            out.append(np.zeros((sa.shape[1], sb.shape[1])))
            continue
        a = np.concatenate([sa[p - 1] for p, _ in pairs], axis=1)
        b = np.concatenate([sb[q - 1] for _, q in pairs], axis=1)
        out.append(a @ b.T)
    return out


def combine(levs, S, weights=None):
    """The epilogue's FP64 sum, smallest level first.  weights: {L: w} replacing 2^(-7 L) (a defect)."""
    V = np.zeros_like(levs[0])
    for L in range(S + 1, 1, -1):
        w = 2.0 ** (-BITS * L) if weights is None or L not in weights else weights[L]
        V = V + levs[L - 2] * w
    return V


def scale(V, alpha, ea, eb, bad_a, bad_b):
    """U = ldexp(fl(alpha V), ea_i + eb_j), NaN in the rows and columns of non-finite operand rows."""
    with np.errstate(over='ignore', invalid='ignore'):
        U = np.ldexp(alpha * V, ea[:, None] + eb[None, :])
    U[bad_a, :] = np.nan
    U[:, bad_b] = np.nan
    return U


def tri_mask(m, n):
    """What a tri = 1 call writes: the 128 x 32 tiles (tm, tn) with 32 tn <= 128 tm + 127."""
    tm = np.arange(m)[:, None] // BM
    tn = np.arange(n)[None, :] // BN
    return tn * BN <= tm * BM + BM - 1


def gemm(A, B, C, alpha, S, overwrite=False, tri=False, defect=None, lev=None):
    """The C the kernel leaves: C (m x n, the old contents; ignored inside the write set when overwriting) updated with
    alpha A B^T through S slices.  lev: precomputed (ea, eb, bad_a, bad_b, levels) (see `operands`)."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    m, n = A.shape[0], B.shape[0]
    if defect == 'b_tile_rows':  # the B tile of tile column 1 read from rows 0..31 instead of 32..63
        assert n >= 2 * BN
        B = B.copy()
        B[BN : 2 * BN] = B[:BN]
    if lev is None or defect is not None:
        shift = None
        if defect == 'row_exponent':
            shift = np.zeros(m, dtype=np.int64)
            shift[0] = 1
        ea, sa, bad_a = split(A, S, shift)
        eb, sb, bad_b = split(B, S)
        drop = ((S, 1),) if defect == 'drop_pair' else ()
        levs = levels(sa, sb, S, drop)
    else:
        ea, eb, bad_a, bad_b, levs = lev
    weights = {S + 1: 2.0 ** (-BITS * (S + 2))} if defect == 'level_weight' else None
    U = scale(combine(levs, S, weights), alpha, ea, eb, bad_a, bad_b)
    C = np.array(C, dtype=np.float64, copy=True)
    if overwrite and defect != 'ignore_overwrite':
        new = U
    else:
        new = C + U
    if defect == 'tile_twice':
        new[:BM, :BN] = new[:BM, :BN] + U[:BM, :BN]
    mask = tri_mask(m, n) if tri else np.ones((m, n), dtype=bool)
    C[mask] = new[mask]
    return C


def operands(A, B, S, product=None):
    """(ea, eb, bad_a, bad_b, levels) for `gemm(lev=...)`.  product(sa, sb, S): the level list computed elsewhere (a
    device matmul for large shapes: any exact integer matmul gives the same levels)."""
    ea, sa, bad_a = split(A, S)
    if B is A:
        eb, sb, bad_b = ea, sa, bad_a
    else:
        eb, sb, bad_b = split(B, S)
    levs = (product or levels)(sa, sb, S)
    return ea, eb, bad_a, bad_b, levs


def method_bound(ea, eb, k, S, alpha=1.0):
    """Componentwise bound on |U - alpha (A B^T)_ij|, U the update before it is added to C, for finite operands whose
    scaled entries x 2^-e stay normal:

        |U_ij - alpha P_ij| <= |alpha| 2^(ea_i + eb_j) k c_S,
        c_S = 2^(-7S-1) (1 + 2^(-7S-1)) + (S - 1) 2^(-7S-2) 128/127 + 0.26 (S + 1) u,  u = 2^-53.

    Per term of the dot product, with a' = a 2^-ea, b' = b 2^-eb (|a'|, |b'| < 1/2) and their S-slice truncations
    alpha_a, alpha_b (remainders |rho| <= 2^(-7S-1)):
      truncation  |a'b' - alpha_a alpha_b| = |a' rho_b + rho_a b' - rho_a rho_b| <= 2^(-7S-1) + 2^(-14S-2);
      dropped     the pairs of levels L = S+2 .. 2S, 2S+1-L of them at level L, each at most 64^2 2^(-7L):
                  sum <= (S - 1) 2^(12 - 7(S+2)) (1 + 2^-7 + ...) = (S - 1) 2^(-7S-2) 128/127;
      rounding    every partial sum of the kept levels is at most k (sum_p 64 2^(-7p))^2 <= 0.254 k; the S - 1
                  additions of the epilogue and fl(alpha V) each add at most u times that.
    The scaling by 2^(ea + eb) is exact while the result stays normal."""
    c = (2.0 ** (-7 * S - 1) * (1 + 2.0 ** (-7 * S - 1)) + (S - 1) * 2.0 ** (-7 * S - 2) * 128 / 127
         + 0.26 * (S + 1) * U64)
    return abs(alpha) * np.ldexp(float(k) * c, (ea[:, None] + eb[None, :]))


def explain(A, B, alpha, S, got, want, i, j):
    """A sentence naming the level or slice pair whose loss or duplication explains got != want at (i, j), if one does."""
    ea, sa, bad_a = split(A[i : i + 1], S)
    eb, sb, bad_b = split(B[j : j + 1], S)
    if bad_a[0] or bad_b[0] or not (np.isfinite(got) and np.isfinite(want)) or alpha == 0:
        return 'no level explains it (non-finite entry)'
    d = np.ldexp((got - want) / alpha, -int(ea[0] + eb[0]))  # the difference in units of the level sum V
    levs = levels(sa, sb, S)
    V = abs(float(combine(levs, S)[0, 0]))
    tol = 4 * (S + 1) * U64 * max(V, 1e-300)
    for L in range(2, S + 2):
        w = float(levs[L - 2][0, 0]) * 2.0 ** (-BITS * L)
        if w != 0 and abs(d + w) <= tol:
            return 'consistent with level %d missing' % L
        if w != 0 and abs(d - w) <= tol:
            return 'consistent with level %d counted twice' % L
        for p, q in level_pairs(S, L):
            wp = float(sa[p - 1, 0] @ sb[q - 1, 0]) * 2.0 ** (-BITS * L)
            if wp != 0 and abs(d + wp) <= tol:
                return 'consistent with slice pair (%d, %d) of level %d missing' % (p, q, L)
    return 'no single level or slice pair explains it (difference %.3g of the level sum %.3g)' % (d, V)


def tiles_of(bad, limit=8):
    """The 128 x 32 tiles (tm, tn) that hold True entries of a bool matrix, up to `limit` of them."""
    rc = np.argwhere(bad)
    t = sorted({(int(r) // BM, int(c) // BN) for r, c in rc[:100000]})
    return t[:limit] + (['...'] if len(t) > limit else [])
