"""Acceptance checks for kernel-matrix assembly (csrc/assemble.cu): K against the oracle, class by class.

Plain functions on NumPy arrays, shared by the GPU tests (tests/test_assemble_classes.py) and by a CPU test that shows
every check can fail (tests/test_assemble_checks.py).  Each check raises AssertionError with a short diagnosis.

`plan` asks the engine (`sgdml_b200_assemble_plan`, host only) which kernel and launch shape a force-force call gets;
`CLASSES` names one shape per routing class and `classes_of` says which classes a plan belongs to.
`assemble_abs_scale` / `ecstr_abs_scale` and `check_K` give a componentwise error bound for every entry of K.
"""

import collections
import ctypes as C

import numpy as np

U = 2.0 ** -53
KB = 1024
H100_SMS = 132  # H100 SXM5; the tests pass the device's own count where the plan depends on it (k_assemble_large)

# ------------------------------------------------------------------------------------------------ plan query
KERNELS = ('k_assemble', 'k_assemble_v4', 'k_assemble_v5', 'k_assemble_large')  # AsmKernel order
Plan = collections.namedtuple('Plan', 'kernel TJ PG n_chunks grid_x smem sym rows_per_launch slab dl_in_smem')


def plan(n_atoms, n_perms, nk, n_colpts, n_rowpts, square, n_sm=H100_SMS):
    """The plan sgdml_b200_assemble_rows would launch under the current sgdml_b200_set_assemble_variant hooks; kernel
    as its name in KERNELS."""
    from sgdml_b200 import _lib

    out = (C.c_int64 * 10)()
    rc = _lib.lib().sgdml_b200_assemble_plan(n_atoms, n_perms, nk, n_colpts, n_rowpts, int(square), n_sm, out)
    _lib.check(rc, 'assemble_plan')
    v = list(out)
    return Plan(KERNELS[v[0]], *v[1:])


def col_shape(cols, n_atoms):
    """(n_colpts, nk) of a sorted column list as the engine counts them: column points touched, and the most atoms of
    one column point with at least one kept column."""
    cols = np.asarray(cols, dtype=np.int64)
    n3 = 3 * n_atoms
    pts, atoms = cols // n3, (cols % n3) // 3
    nk = max(len(np.unique(atoms[pts == j])) for j in np.unique(pts))
    return len(np.unique(pts)), nk


# the routing classes (csrc/assemble.cu asm_plan) and a shape that reaches each: (N, rotors, swaps, M, sig, variant);
# S = 3^rotors 2^swaps (synth.rotor_swap_group); variant is the sgdml_b200_set_assemble_variant hook.  M >= 3
# everywhere, so that a row range can start after the first and end before the last row point.
Case = collections.namedtuple('Case', 'N rot swap M sig variant cls')
CLASSES = {
    'v4_tj8': Case(9, 1, 1, 45, 20, 0, 'v4 TJ=8 PG=S, several CTAs on grid.x, last group clipped'),
    'v4_tj7': Case(12, 1, 2, 11, 30, 0, 'v4 TJ=7'),
    'v4_pgcut_n14': Case(14, 1, 2, 7, 30, 0, 'v4 PG cut to keep two CTAs per SM'),
    'v4_pgcut_n15': Case(15, 1, 2, 6, 30, 0, 'v4 PG cut to keep two CTAs per SM'),
    'v4_tj3': Case(17, 1, 1, 5, 30, 0, 'v4 TJ=3'),
    'v4_tj2': Case(21, 1, 1, 5, 30, 0, 'v4 TJ=2'),
    'v4_tj1': Case(28, 1, 1, 4, 30, 0, 'v4 TJ=1'),
    'v4_z': Case(40, 1, 1, 4, 40, 0, 'v4 TJ=1, grid.z split'),
    'v4_rem_n13': Case(13, 4, 0, 7, 25, 0, 'v4 PG<S with a remainder chunk'),
    'v4_rem_n42': Case(42, 5, 0, 3, 50, 0, 'v4 PG<S with a remainder chunk'),
    'v5_full': Case(60, 1, 1, 3, 50, 0, 'v5 PG=S'),
    'v5_rem_n73': Case(73, 1, 1, 3, 50, 0, 'v5 PG<S with a remainder chunk'),
    'v5_rem_n45': Case(45, 5, 0, 3, 50, 0, 'v5 PG<S with a remainder chunk'),
    'large_smem': Case(100, 2, 0, 3, 50, 0, 'large, delta table in shared memory'),
    'large_gmem': Case(120, 1, 1, 3, 50, 0, 'large, delta table in global memory'),
    'k_tj': Case(9, 1, 1, 20, 20, 2, 'k_assemble (forced) TJ>1'),
    'k_z': Case(40, 1, 1, 4, 40, 2, 'k_assemble (forced) grid.z split'),
    'large_forced': Case(9, 1, 1, 20, 20, 1, 'large (forced) at a small N, CTAs walk several blocks'),
}
# the class with capped slabs needs more blocks than CTAs of a molecule with hundreds of atoms (the nanotube shape,
# N = 370, S = 3, M = 500: 214 CTAs of 10 MB instead of 264), beyond what the oracle can check in a test: its plan is
# only queried.  No test assembles K in this class (tests/test_large_molecules.py runs N = 370 at M <= 4, below the cap)
SLAB_CAPPED = Case(370, 1, 0, 500, 50, 0, 'large, slab-capped grid')
# every class asm_plan can produce; CLASSES and SLAB_CAPPED together must reach each of them
DOCUMENTED = frozenset({
    'v4 TJ=8 PG=S, several CTAs on grid.x, last group clipped',
    'v4 TJ=7',
    'v4 PG cut to keep two CTAs per SM',
    'v4 TJ=3',
    'v4 TJ=2',
    'v4 TJ=1',
    'v4 TJ=1, grid.z split',
    'v4 PG<S with a remainder chunk',
    'v5 PG=S',
    'v5 PG<S with a remainder chunk',
    'large, delta table in shared memory',
    'large, delta table in global memory',
    'large, slab-capped grid',
    'k_assemble (forced) TJ>1',
    'k_assemble (forced) grid.z split',
    'large (forced) at a small N, CTAs walk several blocks',
})


def n_perms(case):
    return 3 ** case.rot * 2 ** case.swap


def classes_of(p, N, S, n_colpts, n_rowpts, n_sm=H100_SMS):
    """The routing classes plan p (of N atoms, S permutations, n_colpts column points, n_rowpts row points) belongs
    to."""
    out = set()
    if p.kernel == 'k_assemble_v4':
        n_tiles = -(-n_colpts // p.TJ)
        if p.TJ == 8 and p.PG == S and p.grid_x >= 2 and n_tiles % 4 != 0:
            out.add('v4 TJ=8 PG=S, several CTAs on grid.x, last group clipped')
        if p.TJ in (7, 3, 2) or (p.TJ == 1 and p.n_chunks == 1):
            out.add('v4 TJ=%d' % p.TJ)
        if p.TJ == 1 and p.n_chunks > 1:
            out.add('v4 TJ=1, grid.z split')
        if S <= 16 and p.PG < S and p.smem <= 110 * KB:
            out.add('v4 PG cut to keep two CTAs per SM')
        if p.PG < S and S % p.PG != 0:
            out.add('v4 PG<S with a remainder chunk')
    elif p.kernel == 'k_assemble_v5':
        if p.PG == S:
            out.add('v5 PG=S')
        elif S % p.PG != 0:
            out.add('v5 PG<S with a remainder chunk')
    elif p.kernel == 'k_assemble':
        if p.TJ > 1:
            out.add('k_assemble (forced) TJ>1')
        if p.n_chunks > 1:
            out.add('k_assemble (forced) grid.z split')
    else:
        out.add('large, delta table in shared memory' if p.dl_in_smem else 'large, delta table in global memory')
        if N <= 64 and n_rowpts * n_colpts > p.grid_x:  # (the default runs v5 or a smaller kernel up to N = 70...82)
            out.add('large (forced) at a small N, CTAs walk several blocks')
        if p.grid_x < min(n_rowpts * n_colpts, 2 * n_sm):
            out.add('large, slab-capped grid')
    return out


# ------------------------------------------------------------------------------------------------ magnitude
def _atom_perms(tril_perms, N):
    """The atom permutations P (S, N) that induce the descriptor permutations tril_perm[d(a, b)] = d(P a, P b): P a is
    the atom that the images of all N - 1 pairs of a share."""
    a, b = np.tril_indices(N, -1)
    S = tril_perms.shape[0]
    P = np.empty((S, N), dtype=np.int64)
    for p in range(S):
        cnt = np.zeros((N, N), dtype=np.int64)
        A, B = a[tril_perms[p]], b[tril_perms[p]]
        for x in (a, b):
            np.add.at(cnt, (x, A), 1)
            np.add.at(cnt, (x, B), 1)
        P[p] = np.argmax(cnt, axis=1) if N > 2 else np.arange(N)
    return P


def _pair_table(g, N):
    """|G| (N, N, 3): |G[a][b]| = |g_d(a,b)|, zero diagonal."""
    a, b = np.tril_indices(N, -1)
    T = np.zeros((N, N, 3))
    T[a, b] = np.abs(g)
    T[b, a] = np.abs(g)
    return T


class _Terms:
    """Per-problem tables of the magnitude functions: x (M, D), g (M, D, 3), the descriptor and atom permutations."""

    def __init__(self, x, g, lin, sig):
        from oracle import desc as odesc

        self.x = np.asarray(x, dtype=np.float64)
        self.g = np.asarray(g, dtype=np.float64)
        self.M, self.D = self.x.shape
        self.N = odesc.n_atoms_from_dim(self.D)
        self.S = len(lin) // self.D
        self.tp = odesc.tril_perms_from_lin(np.asarray(lin), self.S)
        self.P = _atom_perms(self.tp, self.N)
        self.Pinv = np.argsort(self.P, axis=1)
        self.sig = float(sig)
        self.Jabs = np.abs(odesc.d_desc_from_comp(self.g))  # (M, D, 3N)
        self.G = [None] * self.M

    def pair(self, i, j):
        """delta_p = x_i - x_j[perm_p] (S, D) and n_p = sqrt5 |delta_p|."""
        dl = self.x[i][None, :] - self.x[j][self.tp]
        return dl, np.sqrt(5.0) * np.sqrt(np.sum(dl * dl, axis=1))

    def jt_perm(self, j, w):
        """|J_j^(p)|^T w_p for w (S, D) >= 0: sum_d |J_j[perm_p d]| w_p[d] = |J_j|^T w'_p with w'_p[perm_p d] = w_p[d]."""
        wp = np.empty_like(w)
        np.put_along_axis(wp, self.tp, w, axis=1)
        return wp @ self.Jabs[j]

    def table(self, m):
        if self.G[m] is None:
            self.G[m] = _pair_table(self.g[m], self.N)
        return self.G[m]

    def t_abs(self, i, j):
        """|J_i|^T |J_j^(p)| (S, 3N, 3N) from the pair tables: the sub-block (a, b) is |G_i[a][P^-1 b]| (x) |G_j[Pa][b]|,
        plus sum_g |G_i[a][g]| (x) |G_j[Pa][Pg]| where b = P a (each product of the sparse Jacobians is one term)."""
        N, S = self.N, self.S
        Gi, Gj = self.table(i), self.table(j)
        ar = np.arange(N)
        left = Gi[ar[None, :, None], self.Pinv[:, None, :]]  # (S, N, N, 3): [p, a, b] = |G_i[a][P^-1 b]|
        right = Gj[self.P]  # [p, a, b] = |G_j[Pa][b]|
        T = left[..., :, None] * right[..., None, :]  # (S, N, N, 3, 3)
        Gjp = Gj[self.P[:, :, None], self.P[:, None, :]]  # [p, a, g] = |G_j[Pa][Pg]|
        diag = np.einsum('agc,pagk->pack', Gi, Gjp)
        T[np.arange(S)[:, None], ar[None, :], self.P] += diag
        return T.transpose(0, 1, 3, 2, 4).reshape(S, 3 * N, 3 * N)


def assemble_abs_scale(x, g, lin, sig, cols=None, rows=None):
    """Componentwise magnitude of every force-force entry of K (3NM rows, or the block rows of training points
    rows=(m_begin, m_end); the columns cols, default all): entry (r, k) of block (i, j) gets
        sum_p (1 + n_p/sig) [c1_p (|J_i|^T |delta_p|)_r (|J_j^(p)|^T |delta_p|)_k + c2_p (|J_i|^T |J_j^(p)|)_rk],
    delta_p = x_i - x_j[perm_p], n_p = sqrt5 |delta_p|, c1_p = 25 e_p / (3 sig^4), c2_p = 5 (sig^2 + sig n_p) e_p /
    (3 sig^4), e_p = exp(-n_p/sig): the sum K_ij = sum_p c1_p u_p (x) v_p - c2_p J_i^T J_j^(p) (u_p = -J_i^T delta_p,
    v_p = -J_j^(p)T delta_p) with every factor replaced by its absolute value, and each permutation's term weighted
    by 1 + n_p/sig, which covers how an error in n_p moves e_p and c2_p (check_K derives both)."""
    t = _Terms(x, g, lin, sig)
    N, M, S = t.N, t.M, t.S
    n3 = 3 * N
    cols = np.arange(M * n3) if cols is None else np.asarray(cols, dtype=np.int64)
    m0, m1 = (0, M) if rows is None else rows
    out = np.zeros(((m1 - m0) * n3, len(cols)))
    sig = t.sig
    for j in np.unique(cols // n3):
        sel = np.nonzero(cols // n3 == j)[0]
        keep = cols[sel] - j * n3
        for i in range(m0, m1):
            dl, nrm = t.pair(i, j)
            e = np.exp(-nrm / sig)
            w = 1.0 + nrm / sig
            c1 = w * 25.0 * e / (3 * sig ** 4)
            c2 = w * 5.0 * (sig ** 2 + sig * nrm) * e / (3 * sig ** 4)
            ua = np.abs(dl) @ t.Jabs[i]  # (S, 3N)
            va = t.jt_perm(j, np.abs(dl))[:, keep]
            blk = (ua * c1[:, None]).T @ va + np.tensordot(c2, t.t_abs(i, j)[:, :, keep], axes=1)
            out[(i - m0) * n3:(i - m0 + 1) * n3, sel] = blk
    return out


def ecstr_abs_scale(x, g, lin, sig):
    """Componentwise magnitudes of the energy-constraint entries of the (3NM + M)-square matrix of
    oracle.assemble.assemble_E_cstr: (row (M, 3NM), col (3NM, M), ee (M, M)) for K[n + i, blk_j], K[blk_i, n + j] and
    K[n + i, n + j] (n = 3NM):
        K_fe(i, j)_k: sum_p (1 + n_p/sig) c_p (|J_j^(p)|^T |delta_p|)_k,  c_p = 5 (n_p + sig) e_p / (3 sig^3),
                      delta_p = x_i - x_j[perm_p]  (and the column with i and j exchanged),
        K_ee(i, j):   sum_p (1 + n_p/sig) (1 + (n_p/sig)(1 + n_p/(3 sig))) e_p,  delta_p = x_j - x_i[perm_p],
    the oracle's sums with absolute values, each permutation weighted by 1 + n_p/sig as in assemble_abs_scale:
    dc_p/dn = -(n_p/sig) e_p 5/(3 sig^3) and dK_ee/dn = -(n_p/(3 sig^2))(1 + n_p/sig) e_p, both within (1 + n_p/sig)
    times the term's own size per relative error of n_p."""
    t = _Terms(x, g, lin, sig)
    N, M = t.N, t.M
    n3 = 3 * N
    sig = t.sig
    row = np.zeros((M, M * n3))
    ee = np.zeros((M, M))
    for i in range(M):
        for j in range(M):
            dl, nrm = t.pair(i, j)
            e = np.exp(-nrm / sig)
            w = 1.0 + nrm / sig
            cp = w * 5.0 * (nrm + sig) * e / (3 * sig ** 3)
            row[i, j * n3:(j + 1) * n3] = cp @ t.jt_perm(j, np.abs(dl))
            # K[n + j, n + i] takes delta = x_i - x_j[perm] (oracle: diff2 of the pair (j, i))
            ee[j, i] = np.sum(w * (1 + (nrm / sig) * (1 + nrm / (3 * sig))) * e)
    col = np.zeros((M * n3, M))
    for i in range(M):
        col[i * n3:(i + 1) * n3, :] = row[:, i * n3:(i + 1) * n3].T  # K[blk_i, n + j] is K_fe of the pair (j, i)
    return row, col, ee


def ecstr_full_scale(x, g, lin, sig):
    """Magnitudes of the whole (3NM + M)-square energy-constrained matrix."""
    ff = assemble_abs_scale(x, g, lin, sig)
    row, col, ee = ecstr_abs_scale(x, g, lin, sig)
    return np.block([[ff, col], [row, ee]])


# ------------------------------------------------------------------------------------------------ the check
CHECK_C = 8


def n_terms(N, S):
    """k of the bound: the permutations, the descriptor length and twice the atoms."""
    return S + N * (N - 1) // 2 + 2 * N


def tau(k):
    return CHECK_C * k * U


def check_K(K, K_ref, scale, k, what='K', n_atoms=None, cols=None, m_begin=0):
    """|K - K_ref| <= tau scale componentwise, tau = c k u with c = CHECK_C = 8 and k = n_terms(N, S).  Returns
    max |K - K_ref| / (tau scale) for reporting.  n_atoms, cols (the column list of K) and m_begin (its first row
    point) only refine the diagnosis: block (i, j) and entry (r, k) of the first entry outside the bound.

    Derivation of c (u = 2^-53, gamma_n = n u / (1 - n u); every error is relative to the matching term of
    assemble_abs_scale, which dominates the absolute value of every partial sum either side forms):
      * The kernels (k_assemble, v4, v5 and large share the arithmetic): delta = x_i - x_j one rounding; u_p, v_p sum
        N - 1 products each: gamma_N.  |delta_p|^2 sums 2D squares (each pair twice) in any order: gamma_2D relative,
        so n_p = sqrt5 sqrt(n2 / 2) is within (D + 3) u of itself.  e_p = exp(-n_p/sig) adds 2u and moves by
        (n_p/sig) dn/n_p; c1_p, c2_p add 3 roundings each, and (sig^2 + sig n_p) moves by dn/sig relative: c1_p,
        c2_p within (1 + n_p/sig)(D + 3) u + 5u.  T_p: one product (a != P^-1 b) or N - 1 (b = P a): gamma_N.
        c1 u (x) v and c2 T add one rounding each into the accumulator, 2S terms: gamma_2S.  Together
        (1 + n_p/sig) gamma_{2S + D + 2N + 12}.
      * The FP64 oracle: diff one rounding; the norm sums D squares: (D/2 + 2) u in n_p; exp and the factors 6u;
        inner = diff . J_j^(p) and K = J_i^T W have N - 1 non-zero products each (the zeros of the dense Jacobians
        add exactly); W sums 2S terms: (1 + n_p/sig) gamma_{2S + D/2 + 2N + 10}.
    The two sides together stay below (4S + 1.5D + 4N + 22) u <= 4 k u + 22 u for k = S + D + 2N, and k >= 36 for
    every shape tested (N >= 7), so |K - K_ref| <= 5 k u (1 + O(ku)) scale: c = 8 leaves margin for second-order
    terms.  The energy-constraint entries sum N - 1 products per permutation and S permutations (K_fe) or S terms
    (K_ee) with the same factor errors: the same bound.  scale = -1 is exact.  A NaN fails (NaN <= bound is false)."""
    K = np.asarray(K, dtype=np.float64)
    K_ref = np.asarray(K_ref, dtype=np.float64)
    assert K.shape == K_ref.shape == scale.shape, (what, K.shape, K_ref.shape, scale.shape)
    t = tau(k)
    err = np.abs(K - K_ref)
    ok = err <= t * scale
    if not np.all(ok):
        bad = np.argwhere(~ok)
        ratio = np.where(ok, 0.0, err / (t * scale))
        r, c = (int(v) for v in np.unravel_index(int(np.nanargmax(np.where(np.isnan(ratio), np.inf, ratio))), K.shape))
        where = 'entry (%d, %d)' % (r, c)
        if n_atoms is not None:
            n3 = 3 * n_atoms
            col = int(cols[c]) if cols is not None else c
            where = 'block (%d, %d), entry (%d, %d)' % (m_begin + r // n3, col // n3, r % n3, col % n3)
        raise AssertionError(
            '%s: %d entries outside tau = %.2e times the scale; worst at %s: K %r, K_ref %r, |err| / (tau scale) %.3g'
            % (what, bad.shape[0], t, where, float(K[r, c]), float(K_ref[r, c]), float(ratio[r, c]))
        )
    return float(np.max(err / (t * np.maximum(scale, 1e-300))))
