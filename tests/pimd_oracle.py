"""NumPy restatement of the device ring-polymer integrator (k_pimd_step in csrc/md.cu, sgdml_b200_pimd_run): the
normal-mode matrix C, the per-mode tables, the PILE-L BAOAB step and the quantum kinetic-energy estimators, driven by
any force function.

The host constants are computed with the scalar functions of `math` (the C library's, as the engine's host code), the
sums over beads and modes run in index order, and every update rounds as written (NumPy never fuses a multiply and an
add), so with the same forces positions and velocities agree with the device bit for bit.  The noise is
md_oracle.normals with replica index p P + k for mode k of polymer p.
"""

import math

import numpy as np

import md_oracle

THREADS = 128  # MD_THREADS: the order of the device's fixed-order reductions


def normal_modes(P):
    """C (P, P): q_k = sum_j C[j, k] x_j, x_j = sum_k C[j, k] q_k."""
    C = np.empty((P, P))
    for j in range(P):
        for k in range(P):
            if k == 0:
                C[j, k] = math.sqrt(1.0 / P)
            elif 2 * k < P:
                C[j, k] = math.sqrt(2.0 / P) * math.cos(2.0 * math.pi * j * k / P)
            elif 2 * k == P:
                C[j, k] = math.sqrt(1.0 / P) * (-1.0 if j % 2 else 1.0)
            else:
                C[j, k] = math.sqrt(2.0 / P) * math.sin(2.0 * math.pi * j * k / P)
    return C


def constants(P, dt, kT, hbar, gamma, lam, s):
    """The run's constants as the engine's host computes them: h, omega_P, the mode frequencies and tables
    (cos, sin/omega, -omega sin, c1), sigma (P, 3N) and the estimators' constants."""
    s = np.asarray(s, dtype=np.float64)
    dimi = s.shape[0]
    h = 0.5 * dt
    kTP = P * kT
    wP = kTP / hbar
    t = {'h': h, 'kTP': kTP, 'wP': wP, 'C': normal_modes(P), 'w': np.zeros(P), 'cos': np.ones(P),
         'sow': np.full(P, h), 'msin': np.zeros(P), 'c1': np.zeros(P), 'sigma': np.empty((P, dimi))}
    for k in range(P):
        g = gamma
        if k > 0:
            wk = 2.0 * wP * math.sin(math.pi * k / P)
            t['w'][k] = wk
            t['cos'][k] = math.cos(wk * h)
            t['sow'][k] = math.sin(wk * h) / wk
            t['msin'][k] = -wk * math.sin(wk * h)
            g = 2.0 * lam * wk
        c1 = math.exp(-g * dt)
        t['c1'][k] = c1
        t['sigma'][k] = np.sqrt((1.0 - c1 * c1) * kTP * s)
    t['kprim0'] = 0.5 * (dimi * P) * kT
    t['kspring'] = 0.5 * wP * wP / P
    t['kcv0'] = 0.5 * dimi * kT
    t['kvir'] = 0.5 / P
    return t


def to_modes(C, X):
    """X (n_poly, P, 3N) -> (n_poly, P, 3N), summed over beads in order."""
    P = C.shape[0]
    out = np.empty_like(X)
    for k in range(P):
        acc = C[0, k] * X[:, 0]
        for j in range(1, P):
            acc = acc + C[j, k] * X[:, j]
        out[:, k] = acc
    return out


def from_modes(C, Q):
    P = C.shape[0]
    out = np.empty_like(Q)
    for j in range(P):
        acc = C[j, 0] * Q[:, 0]
        for k in range(1, P):
            acc = acc + C[j, k] * Q[:, k]
        out[:, j] = acc
    return out


def free_ring(t, Q, U):
    """A: the exact harmonic rotation of every normal mode over h."""
    c, so, ms = t['cos'][:, None], t['sow'][:, None], t['msin'][:, None]
    return c * Q + so * U, ms * Q + c * U


def thermostat(t, U, xi):
    """O: xi (n_poly, P, 3N) standard normals per mode."""
    return t['c1'][:, None] * U + t['sigma'] * xi


def mode_noise(seed, step, n_poly, P, dimi):
    """xi (n_poly, P, 3N) of global step `step`: md_oracle.normals with replica p P + k for mode k."""
    return md_oracle.normals(seed, step, n_poly * P, dimi).reshape(n_poly, P, dimi)


def _tree(x):
    """The device's sum: x (..., m) spread over THREADS threads (thread t sums x[t], x[t + THREADS], ... in order),
    then a halving tree over the threads."""
    m = x.shape[-1]
    acc = np.zeros(x.shape[:-1] + (THREADS,))
    for i0 in range(0, m, THREADS):
        w = min(THREADS, m - i0)
        acc[..., :w] = acc[..., :w] + x[..., i0:i0 + w]
    w = THREADS // 2
    while w > 0:
        acc = acc[..., :w] + acc[..., w:2 * w]
        w //= 2
    return acc[..., 0]


def kinetic(V, s):
    """Per bead E_kin (n_poly, P) in k_md_step's order: thread t sums the coordinate pairs t, t + THREADS, ..."""
    e = V * V / s
    dimi = e.shape[-1]
    n_pairs = (dimi + 1) // 2
    pairs = np.zeros(e.shape[:-1] + (2 * n_pairs,))
    pairs[..., :dimi] = e  # a missing last coordinate adds 0.0: exact, every term is >= 0
    acc = np.zeros(e.shape[:-1] + (THREADS,))
    for j0 in range(0, n_pairs, THREADS):
        w = min(THREADS, n_pairs - j0)
        for q in (0, 1):
            acc[..., :w] = acc[..., :w] + pairs[..., 2 * j0 + q:2 * (j0 + w):2]
    return 0.5 * _tree(acc)


def estimators(t, X, F, s):
    """K_prim, K_cv (n_poly,) of bead positions X and forces F (n_poly, P, 3N)."""
    P = X.shape[1]
    xb = X[:, 0]
    for j in range(1, P):
        xb = xb + X[:, j]
    xb = xb / P
    spr = np.zeros_like(xb)
    vir = np.zeros_like(xb)
    for j in range(P):
        d = X[:, j] - X[:, (j + 1) % P]
        spr = spr + d * d
        vir = vir + (X[:, j] - xb) * F[:, j]
    spr = _tree(spr / s)
    vir = _tree(vir)
    return t['kprim0'] - t['kspring'] * spr, t['kcv0'] - t['kvir'] * vir


def run(forces, R, V, s, n_steps, dt, kT, hbar, gamma=0.0, lam=0.0, seed=0, step0=0, stride=0, F=None, E=None):
    """PILE-L BAOAB from bead positions and velocities R, V (n_poly, P, 3N) with s (3N,) inverse masses.
    forces(R (n_poly P, 3N)) -> (E (n_poly P,), F).  Returns the final (R, V, F, E) and the frames {'R', 'V' (n_poly,
    P, 3N), 'E_pot', 'E_kin' (n_poly, P), 'K_prim', 'K_cv' (n_poly,)} after every stride-th step."""
    R = np.array(R, dtype=np.float64)
    V = np.array(V, dtype=np.float64)
    n_poly, P, dimi = R.shape
    s = np.asarray(s, dtype=np.float64)
    t = constants(P, dt, kT, hbar, gamma, lam, s)
    h = t['h']

    def ev(R):
        E, F = forces(R.reshape(n_poly * P, dimi))
        return np.asarray(E).reshape(n_poly, P), np.asarray(F).reshape(n_poly, P, dimi)

    if F is None:
        E, F = ev(R)
    use_O = gamma > 0.0 or (lam > 0.0 and P > 1)
    frames = {k: [] for k in ('R', 'V', 'E_pot', 'E_kin', 'K_prim', 'K_cv')}
    for n in range(n_steps):
        V = V + h * (F * s)
        Q, U = to_modes(t['C'], R), to_modes(t['C'], V)
        Q, U = free_ring(t, Q, U)
        if use_O:
            U = thermostat(t, U, mode_noise(seed, step0 + n, n_poly, P, dimi))
        Q, U = free_ring(t, Q, U)
        R, V = from_modes(t['C'], Q), from_modes(t['C'], U)
        E, F = ev(R)
        V = V + h * (F * s)
        if stride and (n + 1) % stride == 0:
            kp, kcv = estimators(t, R, F, s)
            for key, val in (('R', R), ('V', V), ('E_pot', E), ('E_kin', kinetic(V, s)), ('K_prim', kp),
                             ('K_cv', kcv)):
                frames[key].append(np.array(val))
    return (R, V, F, E), {k: np.array(v) for k, v in frames.items()}


def harmonic_value(P, kT, hbar, omega):
    """The exact finite-P mean of <V>, <K_prim> and <K_cv> per degree of freedom of a harmonic oscillator of
    frequency omega: sum_k omega^2 / (2 beta (omega_k^2 + omega^2))."""
    wP = P * kT / hbar
    wk = 2.0 * wP * np.sin(np.pi * np.arange(P) / P)
    return float(np.sum(omega * omega * kT / (2.0 * (wk * wk + omega * omega))))
