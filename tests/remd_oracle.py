"""NumPy restatement of the device replica exchange (csrc/md.cu: k_remd_exchange before k_md_step, sgdml_b200_remd_run)
on md_oracle's BAOAB step: the per-slot sigma, the exchange schedule and pairing, the Philox exchange draw, the swap and
the velocity rule, driven by any force function.

The state here holds full-step velocities w (md_oracle's), where the device holds v = w - h (F s); the device's
v' = lam w - h (F s) is therefore w' = (lam w - h (F s)) + h (F s) here, with the same roundings, so positions,
velocities, walkers and counts agree bit for bit with the device fed the same forces -- as long as every Metropolis
decision does, which needs exp(D) on both sides to fall on the same side of u: `margin` reports the smallest
|u - exp(D)| of the run.
"""

import numpy as np

import md_oracle

EXCHANGE_BIT = 0x80000000  # first counter word of the exchange draw; the O noise's pair indices stay below it


def is_exchange(c, run_start, every):
    """True when the state at step index c of a run that began at run_start is exchanged."""
    return every >= 1 and c > run_start and c % every == 0


def pairs(c, every, n_temps):
    """The lower slots k of the pairs (k, k + 1) attempted on an exchange of the state at c."""
    return list(range((c // every) % 2, n_temps - 1, 2))


def exchange_uniform(seed, k, l, c):
    """u of pair (k, k + 1) of ladder l on the state at c; k, l, c may be arrays (broadcast)."""
    k, l, c = np.broadcast_arrays(*(np.asarray(x, dtype=np.uint64) for x in (k, l, c)))
    ctr = np.stack([k | np.uint64(EXCHANGE_BIT), l, c & np.uint64(0xFFFFFFFF), c >> np.uint64(32)], axis=-1)
    w = md_oracle.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    return md_oracle._uniform53(w[..., 0], w[..., 1])


def tables(kT):
    """beta (n_temps), lam_up, lam_dn (n_temps - 1) as the engine computes them on the host."""
    kT = np.asarray(kT, dtype=np.float64)
    return 1.0 / kT, np.sqrt(kT[1:] / kT[:-1]), np.sqrt(kT[:-1] / kT[1:])


def delta(beta, k, Ea, Eb):
    return (beta[k] - beta[k + 1]) * (Ea - Eb)


def exchange(st, c, every, seed, kT, h, s, stats):
    """The exchange of the state at c, in place.  st: {'R', 'V' (full-step), 'F', 'E', 'walker'}; stats:
    {'n_accepted', 'n_attempted' (n_ladders, n_temps - 1), 'margin'}."""
    n_temps = len(kT)
    beta, up, dn = tables(kT)
    R, V, F, E, W = st['R'], st['V'], st['F'], st['E'], st['walker']
    for l in range(R.shape[0] // n_temps):
        for k in pairs(c, every, n_temps):
            a = l * n_temps + k
            b = a + 1
            d = delta(beta, k, E[a], E[b])
            u = float(exchange_uniform(seed, k, l, c))
            stats['margin'] = min(stats['margin'], abs(u - np.exp(d)))
            stats['n_attempted'][l, k] += 1
            if not (d >= 0.0 or u < np.exp(d)):
                continue
            stats['n_accepted'][l, k] += 1
            ka, kb = h * (F[a] * s), h * (F[b] * s)
            Va = (dn[k] * V[b] - kb) + kb  # configuration b moves down to slot k
            Vb = (up[k] * V[a] - ka) + ka  # configuration a moves up to slot k + 1
            V[a], V[b] = Va, Vb
            for X in (R, F, E, W):
                X[[a, b]] = X[[b, a]]


def run(forces, R, V, s, kT, n_steps, dt, gamma, every, seed=0, step0=0, stride=0, F=None, E=None, walker=None):
    """A replica-exchange run from (R, V) (n_rep, 3N), n_rep = n_ladders len(kT), beginning at step index step0, with
    s (3N,) inverse masses.  forces(R) -> (E (n_rep,), F).  Returns the final {'R', 'V', 'F', 'E', 'walker'}, the
    frames {'R', 'V', 'E_pot', 'E_kin', 'walker'} after every stride-th step, and {'n_accepted', 'n_attempted',
    'margin'}."""
    st = {'R': np.array(R, dtype=np.float64), 'V': np.array(V, dtype=np.float64)}
    n_rep, dimi = st['R'].shape
    n_temps = len(kT)
    s = np.asarray(s, dtype=np.float64)
    if F is None:
        E, F = forces(st['R'])
    st['F'], st['E'] = np.array(F, dtype=np.float64).reshape(n_rep, dimi), np.array(E, dtype=np.float64)
    st['walker'] = np.arange(n_rep, dtype=np.int32) if walker is None else np.array(walker, dtype=np.int32)
    h, c1, _ = md_oracle.constants(dt, gamma, 0.0, s)
    sigma = np.stack([md_oracle.constants(dt, gamma, kT_k, s)[2] for kT_k in kT])[np.arange(n_rep) % n_temps]
    stats = {'n_accepted': np.zeros((n_rep // n_temps, n_temps - 1), dtype=np.int64),
             'n_attempted': np.zeros((n_rep // n_temps, n_temps - 1), dtype=np.int64), 'margin': np.inf}
    frames = {'R': [], 'V': [], 'E_pot': [], 'E_kin': [], 'walker': []}
    for k in range(n_steps):
        c = step0 + k
        V = st['V'] + h * (st['F'] * s)
        R = st['R'] + h * V
        V = c1 * V + sigma * md_oracle.normals(seed, c, n_rep, dimi)
        R = R + h * V
        E, F = forces(R)
        F = np.array(F, dtype=np.float64).reshape(n_rep, dimi)
        st.update(R=R, F=F, E=np.array(E, dtype=np.float64), V=V + h * (F * s))
        if is_exchange(c + 1, step0, every):
            exchange(st, c + 1, every, seed, kT, h, s, stats)
        if stride and (k + 1) % stride == 0:
            for key, val in (('R', st['R']), ('V', st['V']), ('E_pot', st['E']),
                             ('E_kin', md_oracle.kinetic(st['V'], s)), ('walker', st['walker'])):
                frames[key].append(np.array(val))
    return st, {k: np.array(v) for k, v in frames.items()}, stats
