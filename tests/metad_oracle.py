"""NumPy restatement of multiple-walker metadynamics on the device (csrc/md.cu k_metad_bias, sgdml_b200_metad_run): the
collective variables and their gradients, the hill sum in the kernel's order, the bias force, the deposition schedule
and heights, on top of md_oracle's BAOAB step and noise.

Every product, sum and quotient rounds as md.cuh writes it (NumPy never fuses a multiply and an add), so with the same
model forces the device and this restatement differ only where CUDA's exp and atan2 differ from NumPy's in the last
bit.
"""

import numpy as np

import md_oracle

TYPES = {'distance': 0, 'angle': 1, 'dihedral': 2}
MD_THREADS = 128


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def cv_eval(kind, atoms, X):
    """X (n_rep, N, 3) -> s (n_rep,), g (n_rep, n_atoms_of_cv, 3): the CV and its gradient per atom of the CV."""
    r = [X[:, a] for a in atoms]
    if kind == 'distance':
        d = r[1] - r[0]
        s = np.sqrt(_dot(d, d))
        ok = (s != 0.0)[:, None]
        gj = np.where(ok, d / np.where(ok, s[:, None], 1.0), 0.0)
        return s, np.stack([-gj, gj], 1)
    if kind == 'angle':
        a, b = r[0] - r[1], r[2] - r[1]
        c = _cross(a, b)
        cn = np.sqrt(_dot(c, c))
        s = np.arctan2(cn, _dot(a, b))
        ok = (cn != 0.0)[:, None]
        da = np.where(ok, (_dot(a, a) * cn)[:, None], 1.0)
        db = np.where(ok, (_dot(b, b) * cn)[:, None], 1.0)
        gi = np.where(ok, _cross(a, c) / da, 0.0)
        gk = np.where(ok, _cross(c, b) / db, 0.0)
        return s, np.stack([gi, -(gi + gk), gk], 1)
    b1, b2, b3 = r[1] - r[0], r[2] - r[1], r[3] - r[2]
    m, n = _cross(b1, b2), _cross(b2, b3)
    nb = np.sqrt(_dot(b2, b2))
    s = np.arctan2(nb * _dot(b1, n), _dot(m, n))
    mm, nn, bb = _dot(m, m), _dot(n, n), _dot(b2, b2)
    ok = ((mm != 0.0) & (nn != 0.0))[:, None]
    fi = (nb / np.where(ok[:, 0], mm, 1.0))[:, None]
    fl = (nb / np.where(ok[:, 0], nn, 1.0))[:, None]
    p = (_dot(b1, b2) / bb)[:, None]
    q = (_dot(b3, b2) / bb)[:, None]
    gi = -(fi * m)
    gl = fl * n
    t = p * gi - q * gl
    g = np.stack([gi, -(gi + t), t - gl, gl], 1)
    return s, np.where(ok[:, None], g, 0.0)


def wrap(e):
    """a dihedral's hill difference into [-pi, pi) by one step, as the kernel"""
    e = np.asarray(e, dtype=np.float64)
    return np.where(e >= np.pi, e - 2.0 * np.pi, np.where(e < -np.pi, e + 2.0 * np.pi, e))


def block_sum(terms):
    """terms (..., K) in the kernel's order: thread t adds terms t, t + 128, ... from 0.0, then the tree."""
    K = terms.shape[-1]
    pad = (-K) % MD_THREADS
    t = np.concatenate([terms, np.zeros(terms.shape[:-1] + (pad,))], -1)
    t = t.reshape(terms.shape[:-1] + (-1, MD_THREADS))
    part = np.zeros(terms.shape[:-1] + (MD_THREADS,))
    for row in range(t.shape[-2]):
        part = part + t[..., row, :]
    w = MD_THREADS // 2
    while w > 0:
        part = part[..., :w] + part[..., w:2 * w]
        w //= 2
    return part[..., 0]


def hill_sum(s, types, C, W, H):
    """V and dV/ds (n_cv,) of one replica at CVs s over hills C, W (K, n_cv), H (K,) in the kernel's order."""
    a = np.zeros(len(H))
    u = []
    for j, t in enumerate(types):
        e = s[j] - C[:, j]
        if t == 'dihedral':
            e = wrap(e)
        uj = e / W[:, j]
        u.append(uj)
        a = a + uj * uj
    x = H * np.exp(-0.5 * a)
    V = block_sum(x)
    dV = np.array([block_sum(0.0 - x * (u[j] / W[:, j])) for j in range(len(types))])
    return V, dV


def bias(R, cvs, n_walkers, hills):
    """(s (n_rep, n_cv), V (n_rep,), Fb (n_rep, 3N)) of positions R (n_rep, 3N) under hills: a list per group of
    (C, W, H)."""
    n_rep = R.shape[0]
    X = R.reshape(n_rep, -1, 3)
    types = [k for k, _ in cvs]
    sg = [cv_eval(k, a, X) for k, a in cvs]
    s = np.stack([x[0] for x in sg], 1)
    V = np.zeros(n_rep)
    dV = np.zeros((n_rep, len(cvs)))
    for r in range(n_rep):
        C, W, H = hills[r // n_walkers]
        V[r], dV[r] = hill_sum(s[r], types, C, W, H)
    Fb = np.zeros_like(R)
    seen = []
    for _, atoms in cvs:
        for a in atoms:
            if a in seen:
                continue
            seen.append(a)
            fb = np.zeros((n_rep, 3))
            for j, (_, aj) in enumerate(cvs):
                if a in aj:
                    fb = fb - dV[:, j:j + 1] * sg[j][1][:, aj.index(a)]
            Fb[:, 3 * a:3 * a + 3] = fb
    return s, V, Fb, seen


def total_force(Fm, Fb, touched):
    """F = Fm + Fb on the touched atoms (rounded once), Fm elsewhere"""
    F = np.array(Fm)
    for a in touched:
        F[:, 3 * a:3 * a + 3] = Fm[:, 3 * a:3 * a + 3] + Fb[:, 3 * a:3 * a + 3]
    return F


def n_deposits(start, n_steps, pace):
    """#{c in (start, start + n_steps] : c % pace == 0}"""
    return (start + n_steps) // pace - start // pace


def empty_hills(n_groups, n_cv):
    return [(np.zeros((0, n_cv)), np.zeros((0, n_cv)), np.zeros(0)) for _ in range(n_groups)]


def run(forces, R, V, s, cvs, n_walkers, hills, n_steps, dt, gamma=0.0, kT=0.0, w0=0.0, widths=None, pace=1,
        dkT=np.inf, seed=0, step0=0, stride=0):
    """Metadynamics from (R, V) (n_rep, 3N) at step index step0 with s (3N,) inverse masses, the CVs `cvs` (a list of
    (kind, atoms)), n_walkers per group and the groups' committed hills (a list of (C, W, H)).  forces(R) -> (E, Fm).
    Returns (R, V, Fm, E, s_cv, V_bias, hills) after the run and the frames {'R', 'V', 'E_pot', 'E_kin', 'cv', 'bias'}
    after every stride-th step."""
    R = np.array(R, dtype=np.float64)
    V = np.array(V, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    hills = [tuple(np.array(x) for x in g) for g in hills]
    widths = np.asarray(widths if widths is not None else np.ones(len(cvs)), dtype=np.float64)
    E, Fm = forces(R)
    cv, Vb, Fb, touched = bias(R, cvs, n_walkers, hills)
    F = total_force(Fm, Fb, touched)
    h, c1, sigma = md_oracle.constants(dt, gamma, kT, s)
    frames = {k: [] for k in ('R', 'V', 'E_pot', 'E_kin', 'cv', 'bias')}
    for k in range(n_steps):
        c = step0 + k + 1
        V = V + h * (F * s)
        R = R + h * V
        if gamma > 0.0:
            V = c1 * V + sigma * md_oracle.normals(seed, step0 + k, R.shape[0], R.shape[1])
        R = R + h * V
        E, Fm = forces(R)
        cv, Vb, Fb, touched = bias(R, cvs, n_walkers, hills)
        F = total_force(Fm, Fb, touched)
        V = V + h * (F * s)
        if stride and (k + 1) % stride == 0:
            for key, val in (('R', R), ('V', V), ('E_pot', E), ('E_kin', md_oracle.kinetic(V, s)), ('cv', cv),
                             ('bias', Vb)):
                frames[key].append(np.array(val))
        if c % pace == 0:
            ht = w0 * np.exp(-Vb / dkT)
            new = []
            for g, (C, W, H) in enumerate(hills):
                sl = slice(g * n_walkers, (g + 1) * n_walkers)
                new.append((np.concatenate([C, cv[sl]]), np.concatenate([W, np.tile(widths, (n_walkers, 1))]),
                            np.concatenate([H, ht[sl]])))
            hills = new
    return (R, V, Fm, E, cv, Vb, hills), {k: np.array(v) for k, v in frames.items()}
