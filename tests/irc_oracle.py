"""NumPy restatement of the device reaction path (csrc/md.cu k_irc_init / k_irc_step, sgdml_b200_irc_rk4): the mode
check, the start of both branches, the RK4 stages of dx/ds = d(F(x)) in mass-weighted coordinates, the acceptance test
and the path of many saddles, driven by any force function, in the kernels' order and roundings (md.cuh).

Replicas 2k and 2k + 1 of an (n_rep, 3N) array are the forward and backward branch of saddle k.  Every sum is
relax_oracle's block_sum; NumPy never fuses a multiply and an add, so with the same forces the results agree with the
kernels bit for bit.
"""

import numpy as np

from relax_oracle import atom_max2, block_sum

POINT, K1, K2, K3, K4 = 0, 1, 2, 3, 4


def direction(f, r):
    """d = r F / sqrt(sum (r F)^2), 0 when the sum is 0: (3N,) -> (3N,)."""
    g = r * f
    q = block_sum(g * g)
    if q == 0.0:
        return np.zeros_like(g)
    return g / np.sqrt(q)


def init_mode(mode, r):
    """k_irc_init's check: the mass-weighted unit mode, or ValueError for a mode that is not finite or has norm 0."""
    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
        v = np.asarray(mode, dtype=np.float64) / r
        q = block_sum(v * v)
        v = v / np.sqrt(q)
    if not (np.isfinite(q) and q > 0.0):
        raise ValueError('every mode must be finite with a nonzero mass-weighted norm')
    return v


def irc(forces, R0, E0, F0, modes, inv_mass, max_points, step, fmax):
    """sgdml_b200_irc_rk4 from the saddles R0 (n_pairs, 3N) with the energies E0 (n_pairs,) and forces F0 (n_pairs, 3N)
    the handle stored for them, the modes (n_pairs, 3N) and the inverse mass per coordinate inv_mass (3N,); forces(R)
    -> (E (n_rep,), F).  Returns {'R', 'F', 'E' (whole handle, final state), 'R_path' (n_rep, max_points, 3N),
    'E_path' (n_rep, max_points), 'n_points', 'end', 'fmax' (n_rep,)}."""
    R0 = np.asarray(R0, dtype=np.float64)
    n_pairs, dimi = R0.shape
    n_rep = 2 * n_pairs
    r = np.sqrt(np.asarray(inv_mass, dtype=np.float64))
    h = float(step)
    hh, h6 = h / 2.0, h / 6.0
    thr = float(fmax) * float(fmax)
    mp = int(max_points)
    V = np.array([init_mode(modes[k], r) for k in range(n_pairs)]).reshape(n_pairs, dimi)

    Rn = np.repeat(R0, 2, axis=0)
    Fn = np.repeat(np.asarray(F0, dtype=np.float64).reshape(n_pairs, dimi), 2, axis=0)
    E_n = np.repeat(np.asarray(E0, dtype=np.float64).reshape(n_pairs), 2)
    R = np.empty_like(Rn)
    R[0::2] = R0 + r * (h * V)
    R[1::2] = R0 + r * ((-h) * V)
    R_path = np.full((n_rep, mp, dimi), np.nan)
    E_path = np.full((n_rep, mp), np.nan)
    R_path[:, 0] = Rn
    E_path[:, 0] = E_n
    K = np.zeros((n_rep, dimi))
    phase = np.full(n_rep, POINT)
    end = np.zeros(n_rep, dtype=np.int32)
    n_points = np.ones(n_rep, dtype=np.int64)
    f2 = np.zeros(n_rep)

    def launch(b, F, E, advance):
        if end[b]:
            return
        if phase[b] == POINT:
            if not (E[b] < E_n[b]):
                R[b], F[b], E[b] = Rn[b], Fn[b], E_n[b]
                f2[b] = atom_max2(Fn[b])
                end[b] = 2
            else:
                n = n_points[b]
                Rn[b], Fn[b] = R[b], F[b]
                R_path[b, n], E_path[b, n] = R[b], E[b]
                n_points[b] = n + 1
                E_n[b] = E[b]
                f2[b] = atom_max2(F[b])
                end[b] = 1 if f2[b] < thr else (3 if n_points[b] == mp else 0)
            phase[b] = K1
        if end[b] or not advance:
            return
        d = direction(F[b], r)
        ph = phase[b]
        c = h if ph == K3 else (h6 if ph == K4 else hh)
        x = d
        if ph == K1:
            K[b] = d
        elif ph == K4:
            x = K[b] + d
        else:
            K[b] = K[b] + 2.0 * d
        R[b] = Rn[b] + r * (c * x)
        phase[b] = POINT if ph == K4 else ph + 1

    def evaluate():
        E, F = forces(R)
        return np.array(E, dtype=np.float64).reshape(n_rep), np.array(F, dtype=np.float64).reshape(R.shape)

    E, F = evaluate()
    for _ in range(4 * (mp - 1)):
        for b in range(n_rep):
            launch(b, F, E, True)
        if np.all(end != 0):
            break
        E, F = evaluate()
    else:
        for b in range(n_rep):
            launch(b, F, E, False)
    return {'R': R, 'F': F, 'E': E, 'R_path': R_path, 'E_path': E_path, 'n_points': n_points, 'end': end,
            'fmax': np.sqrt(f2)}
