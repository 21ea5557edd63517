"""NumPy restatement of umbrella sampling with replica exchange on the device (csrc/md.cu k_umbrella_bias,
k_umbrella_exchange, sgdml_b200_umbrella_run): the harmonic window restraints on metad_oracle's CVs, their bias force,
the Hamiltonian exchange (schedule, Philox draw, decision, moved rows, velocity correction, frames) on md_oracle's BAOAB
step and noise; and a plain NumPy MBAR, independent of the device's reduction order.

The state here holds full-step velocities w (md_oracle's), where the device holds v = w - h (F s); an accepted swap
stores v' = w - h (F_new s) on the device, which is w' = (w - h (F_new s)) + h (F_new s) here, with the same
roundings.  Every product and sum rounds as md.cuh writes it, so with the same model forces the device and this
restatement differ only where CUDA's exp and atan2 differ from NumPy's in the last bit.
"""

import numpy as np
from scipy.special import logsumexp

import md_oracle
import metad_oracle
import remd_oracle


def restraint(s, types, c, kappa):
    """b (n,) and u = db/ds (n, n_cv) of CVs s (n, n_cv) under one window (c, kappa (n_cv,)), in the kernel's order."""
    s = np.asarray(s, dtype=np.float64).reshape(-1, len(types))
    b = np.zeros(s.shape[0])
    u = np.zeros_like(s)
    for j, t in enumerate(types):
        e = s[:, j] - c[j]
        if t == 'dihedral':
            e = metad_oracle.wrap(e)
        u[:, j] = kappa[j] * e
        b = b + (0.5 * u[:, j]) * e
    return b, u


def bias(R, cvs, C, Kap, windows):
    """(s (n_rep, n_cv), b (n_rep,), Fb (n_rep, 3N), touched atoms) of positions R (n_rep, 3N), replica r under window
    windows[r] of the table C, Kap (n_windows, n_cv)."""
    n_rep = R.shape[0]
    X = R.reshape(n_rep, -1, 3)
    types = [k for k, _ in cvs]
    sg = [metad_oracle.cv_eval(k, a, X) for k, a in cvs]
    s = np.stack([x[0] for x in sg], 1)
    b = np.zeros(n_rep)
    u = np.zeros((n_rep, len(cvs)))
    for r in range(n_rep):
        k = windows[r]
        b[r:r + 1], u[r:r + 1] = restraint(s[r], types, C[k], Kap[k])
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
                    fb = fb - u[:, j:j + 1] * sg[j][1][:, aj.index(a)]
            Fb[:, 3 * a:3 * a + 3] = fb
    return s, b, Fb, seen


def slot_windows(n_rep, n_windows):
    return np.arange(n_rep) % n_windows


def evaluate(st, forces, cvs, C, Kap):
    """the state's model E, Fm, its CVs, restraints, Fb and F = Fm + Fb in the slots' windows"""
    E, Fm = forces(st['R'])
    st['E'], st['Fm'] = np.array(E, dtype=np.float64), np.array(Fm, dtype=np.float64).reshape(st['R'].shape)
    reslot(st, cvs, C, Kap)


def reslot(st, cvs, C, Kap):
    st['cv'], st['bias'], Fb, touched = bias(st['R'], cvs, C, Kap, slot_windows(len(st['R']), len(C)))
    st['Fb'] = Fb
    st['F'] = metad_oracle.total_force(st['Fm'], Fb, touched)


def exchange(st, c, every, seed, beta, h, s, cvs, C, Kap, stats):
    """The exchange of the state at c, in place.  st: {'R', 'V' (full-step), 'Fm', 'F', 'E', 'cv', 'bias', 'walker'};
    stats: {'n_accepted', 'n_attempted' (n_ladders, n_windows - 1), 'margin'}."""
    nw = len(C)
    types = [k for k, _ in cvs]
    R = st['R']
    for l in range(R.shape[0] // nw):
        moved = []
        for k in remd_oracle.pairs(c, every, nw):
            a, b = l * nw + k, l * nw + k + 1
            sa, sb = st['cv'][a], st['cv'][b]
            od = restraint(sa, types, C[k], Kap[k])[0][0] + restraint(sb, types, C[k + 1], Kap[k + 1])[0][0]
            nd = restraint(sb, types, C[k], Kap[k])[0][0] + restraint(sa, types, C[k + 1], Kap[k + 1])[0][0]
            d = -(beta * (nd - od))
            u = float(remd_oracle.exchange_uniform(seed, k, l, c))
            stats['margin'] = min(stats['margin'], abs(u - np.exp(d)))
            stats['n_attempted'][l, k] += 1
            if not (d >= 0.0 or u < np.exp(d)):
                continue
            stats['n_accepted'][l, k] += 1
            for key in ('R', 'V', 'Fm', 'E', 'cv', 'walker'):
                X = st[key]
                X[[a, b]] = X[[b, a]]
            moved.append((a, b))
        if moved:
            reslot(st, cvs, C, Kap)
            for a, b in moved:
                for r in (a, b):
                    kn = h * (st['F'][r] * s)
                    st['V'][r] = (st['V'][r] - kn) + kn


def run(forces, R, V, s, cvs, C, Kap, n_steps, dt, gamma=0.0, kT=0.0, every=0, seed=0, step0=0, stride=0,
        walker=None):
    """An umbrella run from (R, V) (n_rep, 3N), n_rep = n_ladders n_windows, at step index step0 with s (3N,) inverse
    masses and the window table C, Kap (n_windows, n_cv).  forces(R) -> (E, Fm).  Returns the final state, the frames
    {'R', 'V', 'E_pot', 'E_kin', 'cv', 'bias', 'walker'} after every stride-th step and the exchange statistics."""
    st = {'R': np.array(R, dtype=np.float64), 'V': np.array(V, dtype=np.float64)}
    n_rep, dimi = st['R'].shape
    nw = len(C)
    s = np.asarray(s, dtype=np.float64)
    st['walker'] = np.arange(n_rep, dtype=np.int32) if walker is None else np.array(walker, dtype=np.int32)
    evaluate(st, forces, cvs, C, Kap)
    h, c1, sigma = md_oracle.constants(dt, gamma, kT, s)
    beta = 1.0 / kT if kT > 0.0 else 0.0
    stats = {'n_accepted': np.zeros((n_rep // nw, nw - 1), dtype=np.int64),
             'n_attempted': np.zeros((n_rep // nw, nw - 1), dtype=np.int64), 'margin': np.inf}
    frames = {k: [] for k in ('R', 'V', 'E_pot', 'E_kin', 'cv', 'bias', 'walker')}
    for k in range(n_steps):
        c = step0 + k
        Vh = st['V'] + h * (st['F'] * s)
        st['R'] = st['R'] + h * Vh
        if gamma > 0.0:
            Vh = c1 * Vh + sigma * md_oracle.normals(seed, c, n_rep, dimi)
        st['R'] = st['R'] + h * Vh
        evaluate(st, forces, cvs, C, Kap)
        st['V'] = Vh + h * (st['F'] * s)
        if remd_oracle.is_exchange(c + 1, step0, every):
            exchange(st, c + 1, every, seed, beta, h, s, cvs, C, Kap, stats)
        if stride and (k + 1) % stride == 0:
            for key, val in (('R', st['R']), ('V', st['V']), ('E_pot', st['E']), ('E_kin', md_oracle.kinetic(st['V'], s)),
                             ('cv', st['cv']), ('bias', st['bias']), ('walker', st['walker'])):
                frames[key].append(np.array(val))
    return st, {k: np.array(v) for k, v in frames.items()}, stats


def mbar(u_kn, N_k, tol=1e-10, max_iter=10000):
    """Plain self-consistent MBAR (Shirts & Chodera 2008, eq. 11) on the reduced potentials u_kn (K, n) of samples
    pooled with N_k (K,) per window: (f (K,) with f_0 = 0, log w (n,) normalised, iterations)."""
    u_kn = np.asarray(u_kn, dtype=np.float64)
    N_k = np.asarray(N_k, dtype=np.float64)
    with np.errstate(divide='ignore'):
        lnN = np.log(N_k)
    f = np.zeros(len(N_k))
    it = 0
    for it in range(1, max_iter + 1):
        L = logsumexp(lnN[:, None] + f[:, None] - u_kn, axis=0)
        fn = -logsumexp(-u_kn - L[None], axis=1)
        fn = fn - fn[0]
        d = np.max(np.abs(fn - f))
        f = fn
        if d < tol:
            break
    L = logsumexp(lnN[:, None] + f[:, None] - u_kn, axis=0)
    return f, -L - logsumexp(-L), it
