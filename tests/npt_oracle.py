"""NumPy restatement of the device NPT step (csrc/md.cu: k_npt_step, sgdml_b200_npt_run) on md_oracle's BAOAB step:
the instantaneous pressure, the barostat's volume move with its own Philox stream, the isotropic rescaling and the
cells, driven by any force function that also returns the virial.

The kinetic energy is summed in the device's order (kinetic below), and every update rounds as the device's, so with
the same forces, virials and transcendental functions the two agree bit for bit.  exp, log and cos may differ from the
device's in the last bit, which the barostat carries into the positions, so device trajectories are compared within a
tolerance.
"""

import numpy as np

import md_oracle

BARO_WORD = 0xFFFFFFFF  # first counter word of the barostat draw: above every O pair index and exchange word
THREADS = 128  # MD_THREADS


def barostat_normal(seed, rep, n):
    """eta of replica rep on the step at counter n (broadcast)."""
    rep, n = np.broadcast_arrays(np.asarray(rep, dtype=np.uint64), np.asarray(n, dtype=np.uint64))
    ctr = np.stack([np.full_like(rep, BARO_WORD), rep, n & np.uint64(0xFFFFFFFF), n >> np.uint64(32)], axis=-1)
    u = md_oracle.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    ua, ub = md_oracle._uniform53(u[..., 0], u[..., 1]), md_oracle._uniform53(u[..., 2], u[..., 3])
    return np.sqrt(-2.0 * np.log(ua)) * np.cos(2.0 * np.pi * ub)


def kinetic(V, s):
    """1/2 sum_i v_i^2 / s_i per replica in k_md_step's E_kin order: thread t adds the coordinates of its pairs
    j = t, t + 128, ... in increasing order, then the tree red[t] += red[t + w] for w = 64, ..., 1."""
    V = np.asarray(V, dtype=np.float64)
    t = V * V / s
    n_rep, dimi = t.shape
    part = np.zeros((n_rep, THREADS))
    n_pairs = (dimi + 1) // 2
    for j0 in range(0, n_pairs, THREADS):
        for q in range(2):
            idx = 2 * np.arange(j0, min(j0 + THREADS, n_pairs)) + q
            idx = idx[idx < dimi]
            part[:, (idx - q) // 2 - j0] = part[:, (idx - q) // 2 - j0] + t[:, idx]
    w = THREADS // 2
    while w > 0:
        part[:, :w] = part[:, :w] + part[:, w:2 * w]
        w //= 2
    return 0.5 * part[:, 0]


def det3(a):
    """|det| of (..., 9) row-major cells, in the host's order (md.cu, npt_parse)."""
    a = np.moveaxis(np.asarray(a, dtype=np.float64), -1, 0)
    return np.abs(a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) +
                  a[2] * (a[3] * a[7] - a[4] * a[6]))


def constants(dt, kT, P0, beta_T, tau_p):
    """c_a, c_b as the engine computes them on the host."""
    rate = beta_T / tau_p
    return rate * dt, 2.0 * kT * rate * dt


def pressure(K, W, V0, eps):
    vol = V0 * np.exp(eps)
    return (2.0 * K + ((W[:, 0] + W[:, 4]) + W[:, 8])) / (3.0 * vol)


def cells(L0, L0inv, eps):
    """The cells a L0 and inverses L0^-1 / a, a = exp(eps / 3), (n_rep, 9) each."""
    a = np.exp(np.asarray(eps) / 3.0)[:, None]
    return a * L0, L0inv / a


def run(forces, R, V, s, L0, L0inv, n_steps, dt, gamma, kT, P0, beta_T, tau_p, seed=0, step0=0, stride=0, eps=None,
        state=None):
    """An NPT run from (R, V) (n_rep, 3N) with s (3N,) inverse masses and base cells L0, L0inv (n_rep, 9), eps the
    log volume ratios (None: 0).  forces(R, cells, cell_invs) -> (E (n_rep,), F (n_rep, 3N), W (n_rep, 9)).  state:
    (E, F, W) of the start (None: evaluated).  Returns the final {'R', 'V', 'F', 'E', 'W', 'eps'} and the frames
    {'R', 'V', 'E_pot', 'E_kin', 'cell', 'P'} after every stride-th step."""
    R = np.array(R, dtype=np.float64)
    V = np.array(V, dtype=np.float64)
    L0 = np.asarray(L0, dtype=np.float64)
    L0inv = np.asarray(L0inv, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    n_rep, dimi = R.shape
    V0 = det3(L0)
    eps = np.zeros(n_rep) if eps is None else np.array(eps, dtype=np.float64)
    E, F, W = forces(R, *cells(L0, L0inv, eps)) if state is None else state
    h, c1, sigma = md_oracle.constants(dt, gamma, kT, s)
    c_a, c_b = constants(dt, kT, P0, beta_T, tau_p)
    reps = np.arange(n_rep)
    frames = {'R': [], 'V': [], 'E_pot': [], 'E_kin': [], 'cell': [], 'P': []}
    for k in range(n_steps):
        c = step0 + k
        pint = pressure(kinetic(V, s), W, V0, eps)
        de = -c_a * (P0 - pint)
        if c_b != 0.0:
            de = de + np.sqrt(c_b / (V0 * np.exp(eps))) * barostat_normal(seed, reps, c)
        mu = np.exp(de / 3.0)[:, None]
        V = V + h * (F * s)
        R = R + h * V
        if gamma > 0.0:
            V = c1 * V + sigma * md_oracle.normals(seed, c, n_rep, dimi)
        R = R + h * V
        R = R * mu
        V = V / mu
        eps = eps + de
        E, F, W = forces(R, *cells(L0, L0inv, eps))
        V = V + h * (F * s)
        if stride and (k + 1) % stride == 0:
            K = kinetic(V, s)
            for key, val in (('R', R), ('V', V), ('E_pot', E), ('E_kin', K), ('cell', cells(L0, L0inv, eps)[0]),
                             ('P', pressure(K, W, V0, eps))):
                frames[key].append(np.array(val))
    final = {'R': R, 'V': V, 'F': F, 'E': E, 'W': W, 'eps': eps}
    return final, {k: np.array(v) for k, v in frames.items()}
