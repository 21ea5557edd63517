"""NumPy restatement of the device optimisers (csrc/md.cu k_fire_step / k_lbfgs_step, sgdml_b200_relax_*): FIRE and
L-BFGS of many replicas, driven by any force function, with the kernels' summation order and roundings (md.cuh).

Every dot product is `block_sum`: 128 per-thread partials over coordinates t, t + 128, ... in order, then a fixed
tree.  NumPy never fuses a multiply and an add, so with the same forces the results agree bit for bit.
"""

import numpy as np

THREADS = 128
FIRE_NMIN, FIRE_FINC, FIRE_FDEC, FIRE_ALPHA0, FIRE_FALPHA = 5, 1.1, 0.5, 0.1, 0.99


def block_sum(x):
    """Sum over the last axis in the kernels' order: (..., n) -> (...)."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[-1]
    k = -(-n // THREADS)
    pad = np.zeros(x.shape[:-1] + (k * THREADS,))
    pad[..., :n] = x  # adding 0.0 to a partial changes nothing
    rows = pad.reshape(x.shape[:-1] + (k, THREADS))
    red = np.zeros(x.shape[:-1] + (THREADS,))
    for j in range(k):
        red = red + rows[..., j, :]
    w = THREADS // 2
    while w > 0:
        red = red[..., :w] + red[..., w:2 * w]
        w //= 2
    return red[..., 0]


def atom_max2(x):
    """max over atoms of (x0 x0 + x1 x1) + x2 x2 per replica, NaN if any is NaN: (..., 3N) -> (...)."""
    x = np.asarray(x, dtype=np.float64)
    a = x.reshape(x.shape[:-1] + (x.shape[-1] // 3, 3))
    return np.max((a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1]) + a[..., 2] * a[..., 2], axis=-1)


def _eval(forces, R):
    E, F = forces(R)
    return np.asarray(E, dtype=np.float64).reshape(R.shape[0]), np.asarray(F, dtype=np.float64).reshape(R.shape)


def _result(R, F, E, n_steps, conv, f2, tested, **extra):
    """'tested': every max_a |F_a| the convergence test compared with fmax, flattened (to keep thresholds off ties)."""
    out = {'R': R, 'F': F, 'E': E, 'n_steps': n_steps, 'converged': conv, 'fmax': np.sqrt(f2),
           'tested': np.concatenate(tested)}
    out.update(extra)
    return out


def fire(forces, R, max_steps, fmax, maxstep, dt, dtmax, E=None, F=None):
    """FIRE from R (n_rep, 3N); forces(R) -> (E (n_rep,), F).  Returns {'R', 'F', 'E', 'n_steps', 'converged', 'fmax',
    'dt', 'alpha', 'n_pos', 'V'} after at most max_steps steps (the replays stop once every replica has converged, which
    changes nothing)."""
    R = np.array(R, dtype=np.float64)
    if F is None:
        E, F = _eval(forces, R)
    n = R.shape[0]
    V = np.zeros_like(R)
    dts = np.full(n, float(dt))
    alpha = np.full(n, FIRE_ALPHA0)
    n_pos = np.zeros(n, dtype=np.int64)
    n_steps = np.zeros(n, dtype=np.int64)
    conv = np.zeros(n, dtype=bool)
    f2 = np.zeros(n)
    thr = fmax * fmax
    tested = []
    for _ in range(max_steps):
        act = ~conv
        f2[act] = atom_max2(F[act])
        tested.append(np.sqrt(f2[act]))
        conv[act] = f2[act] < thr
        act = ~conv
        if not act.any():
            break
        later = act & (n_steps > 0)
        P = block_sum(F * V)
        mix = later & (P > 0.0)
        rst = later & ~(P > 0.0)
        if mix.any():
            vv, ff = block_sum(V[mix] * V[mix]), block_sum(F[mix] * F[mix])
            c = alpha[mix] * (np.sqrt(vv) / np.sqrt(ff))
            om = 1.0 - alpha[mix]
            V[mix] = om[:, None] * V[mix] + c[:, None] * F[mix]
            grow = mix & (n_pos > FIRE_NMIN)
            dts[grow] = np.minimum(dts[grow] * FIRE_FINC, dtmax)
            alpha[grow] = alpha[grow] * FIRE_FALPHA
            n_pos[mix] += 1
        V[rst] = 0.0
        alpha[rst] = FIRE_ALPHA0
        dts[rst] = dts[rst] * FIRE_FDEC
        n_pos[rst] = 0
        V[act] = V[act] + dts[act, None] * F[act]
        dr = dts[act, None] * V[act]
        nrm = np.sqrt(block_sum(dr * dr))
        cap = nrm > maxstep
        dr[cap] = (maxstep * dr[cap]) / nrm[cap, None]
        R[act] = R[act] + dr
        n_steps[act] += 1
        E, F = _eval(forces, R)
    act = ~conv
    f2[act] = atom_max2(F[act])
    tested.append(np.sqrt(f2[act]))
    conv[act] = f2[act] < thr
    return _result(R, F, E, n_steps, conv, f2, tested, dt=dts, alpha=alpha, n_pos=n_pos, V=V)


def lbfgs(forces, R, max_steps, fmax, maxstep, memory, h0, E=None, F=None):
    """L-BFGS from R (n_rep, 3N); forces(R) -> (E (n_rep,), F).  Returns {'R', 'F', 'E', 'n_steps', 'converged',
    'fmax', 'n_hist'}, 'n_hist' (n_steps_run, n_rep) being the pairs each replica used for each step's direction (-1:
    no step)."""
    R = np.array(R, dtype=np.float64)
    if F is None:
        E, F = _eval(forces, R)
    n, dimi = R.shape
    m = int(memory)
    S = np.zeros((n, m, dimi))
    Y = np.zeros((n, m, dimi))
    rho = np.zeros((n, m))
    gamma = np.zeros(n)
    E_prev = np.zeros(n)
    r_prev = np.zeros_like(R)
    g_prev = np.zeros_like(R)
    n_hist = np.zeros(n, dtype=np.int64)
    head = np.zeros(n, dtype=np.int64)
    n_steps = np.zeros(n, dtype=np.int64)
    conv = np.zeros(n, dtype=bool)
    f2 = np.zeros(n)
    thr = fmax * fmax
    trace = []
    tested = []
    for _ in range(max_steps):
        act = ~conv
        f2[act] = atom_max2(F[act])
        tested.append(np.sqrt(f2[act]))
        conv[act] = f2[act] < thr
        if conv.all():
            break
        used = np.full(n, -1)
        R_new = R.copy()
        for b in np.flatnonzero(~conv):
            r, f, e = R[b], F[b], E[b]
            g = -f
            if n_steps[b] > 0:
                slot = (head[b] + 1) % m
                s, y = r - r_prev[b], g - g_prev[b]
                S[b, slot], Y[b, slot] = s, y
                sy, yy = block_sum(s * y), block_sum(y * y)
                if sy > 0.0:
                    head[b] = slot
                    n_hist[b] = min(n_hist[b] + 1, m)
                    gamma[b] = sy / yy
                    rho[b, slot] = 1.0 / sy
                else:
                    n_hist[b] = 0
                if e > E_prev[b]:
                    n_hist[b] = 0
            nh = int(n_hist[b])
            slots = [(head[b] - k) % m for k in range(nh)]
            q = g.copy()
            a = np.zeros(nh)
            for k, sl in enumerate(slots):
                a[k] = rho[b, sl] * block_sum(S[b, sl] * q)
                q = q - a[k] * Y[b, sl]
            z = (gamma[b] if nh > 0 else h0) * q
            for k in range(nh - 1, -1, -1):
                sl = slots[k]
                bk = rho[b, sl] * block_sum(Y[b, sl] * z)
                z = z + S[b, sl] * (a[k] - bk)
            d = -z
            if not (block_sum(d * g) < 0.0):
                n_hist[b] = 0
                d = h0 * f
            L = np.sqrt(atom_max2(d))
            if L > maxstep:
                d = d * (maxstep / L)
            used[b] = n_hist[b]
            r_prev[b], g_prev[b], E_prev[b] = r, g, e
            R_new[b] = r + d
            n_steps[b] += 1
        trace.append(used)
        R = R_new
        E, F = _eval(forces, R)
    act = ~conv
    f2[act] = atom_max2(F[act])
    tested.append(np.sqrt(f2[act]))
    conv[act] = f2[act] < thr
    return _result(R, F, E, n_steps, conv, f2, tested, n_hist=np.array(trace).reshape(-1, n))
