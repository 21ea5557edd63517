"""NumPy restatement of the device dimer search (csrc/md.cu k_dimer_init / k_dimer_step, sgdml_b200_dimer_fire): the
initial projection, the test, the rotation with its curvature fit, the rigid projection and the FIRE translation of
many dimers, driven by any force function, in the kernels' order and roundings (md.cuh).

Replica 2d of an (n_rep, 3N) array is the centre of dimer d and replica 2d + 1 its image.  Every sum is relax_oracle's
block_sum; NumPy never fuses a multiply and an add, so with the same forces the results agree with the kernels bit for
bit.  project: 'rigid' (free molecules), 'translations' (periodic models) or 'none' (test surfaces in the plane only;
the device always projects).
"""

import math

import numpy as np

import relax_oracle
from relax_oracle import atom_max2, block_sum

EVAL_N, TRIAL = 0, 1


def _comp_sums(x):
    """Component sums: block_sum of x with the other components masked to 0.0, (3N,) -> (3,)."""
    c = np.arange(x.shape[-1]) % 3
    return np.array([block_sum(np.where(c == k, x, 0.0)) for k in range(3)])


def _atom_sum(t):
    """Atom sum: block_sum of the (3N,) vector holding t_a at coordinate 3a and 0.0 elsewhere."""
    v = np.zeros(3 * len(t))
    v[0::3] = t
    return block_sum(v)


def _cross(a, b):
    """(..., 3) x (..., 3), md.cuh's cross rounded as written."""
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def project(n, r, project='rigid'):
    """md.cuh 5: the mode n (3N,) at centre r (3N,) without rigid motions, normalised -> (unit mode, its n.n before
    the normalisation)."""
    n = np.array(n, dtype=np.float64)
    r = np.asarray(r, dtype=np.float64)
    if project not in ('rigid', 'translations', 'none'):
        raise ValueError(project)
    if project != 'none':
        na = float(len(n) // 3)
        m = _comp_sums(n) / na
        rb = _comp_sums(r) / na
        n = n - np.tile(m, len(n) // 3)
        if project == 'rigid':
            x = r.reshape(-1, 3) - rb
            l = _cross(x, n.reshape(-1, 3))
            L = [_atom_sum(l[:, c]) for c in range(3)]
            x00, x11, x22 = x[:, 0] * x[:, 0], x[:, 1] * x[:, 1], x[:, 2] * x[:, 2]
            I00, I11, I22 = _atom_sum(x11 + x22), _atom_sum(x00 + x22), _atom_sum(x00 + x11)
            I01, I02, I12 = (-_atom_sum(x[:, a] * x[:, b]) for a, b in ((0, 1), (0, 2), (1, 2)))
            A00 = I11 * I22 - I12 * I12
            A01 = I02 * I12 - I01 * I22
            A02 = I01 * I12 - I11 * I02
            A11 = I00 * I22 - I02 * I02
            A12 = I01 * I02 - I00 * I12
            A22 = I00 * I11 - I01 * I01
            det = (I00 * A00 + I01 * A01) + I02 * A02
            tr = ((I00 + I11) + I22) / 3.0
            if det > 1e-10 * ((tr * tr) * tr):
                w = np.array([((A00 * L[0] + A01 * L[1]) + A02 * L[2]) / det,
                              ((A01 * L[0] + A11 * L[1]) + A12 * L[2]) / det,
                              ((A02 * L[0] + A12 * L[1]) + A22 * L[2]) / det])
                n = n - _cross(np.broadcast_to(w, x.shape), x).ravel()
    nn = block_sum(n * n)
    with np.errstate(divide='ignore', invalid='ignore'):  # a zero mode becomes NaN, as on the device
        return n / np.sqrt(nn), nn


def init_mode(src, r, project_='rigid'):
    """k_dimer_init for one dimer: the unit mode, or ValueError for a mode that is not finite or (almost) rigid."""
    src = np.asarray(src, dtype=np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        n0 = block_sum(src * src)
        n, n1 = project(src, r, project_)
    if not (np.isfinite(n0) and n1 > 1e-12 * n0):
        raise ValueError('every mode must be finite and not (almost) a rigid motion')
    return n


class _Fire(object):
    """One vector's RelaxState for fire_update (md.cu), restated."""

    def __init__(self):
        self.dt = self.alpha = 0.0
        self.n_pos = self.n_steps = 0

    def update(self, r, v, f, dt0, dtmax, maxstep):
        """One FIRE step of r and v (1-D, in place) with force f."""
        if self.n_steps == 0:
            self.dt, self.alpha, self.n_pos = dt0, relax_oracle.FIRE_ALPHA0, 0
        else:
            fv = block_sum(f * v)
            if fv > 0.0:
                vv, ff = block_sum(v * v), block_sum(f * f)
                c = self.alpha * (math.sqrt(vv) / math.sqrt(ff))
                v[:] = (1.0 - self.alpha) * v + c * f
                if self.n_pos > relax_oracle.FIRE_NMIN:
                    self.dt = min(self.dt * relax_oracle.FIRE_FINC, dtmax)
                    self.alpha = self.alpha * relax_oracle.FIRE_FALPHA
                self.n_pos += 1
            else:
                v[:] = 0.0
                self.alpha = relax_oracle.FIRE_ALPHA0
                self.dt = self.dt * relax_oracle.FIRE_FDEC
                self.n_pos = 0
        v[:] = v + self.dt * f
        dr = self.dt * v
        nrm = math.sqrt(block_sum(dr * dr))
        if nrm > maxstep:
            dr = (maxstep * dr) / nrm
        r[:] = r + dr
        self.n_steps += 1


def search(forces, R, modes, max_steps, fmax, separation, cos_trial, sin_trial, rot_min, maxstep, dt, dtmax,
           project_='rigid'):
    """sgdml_b200_dimer_fire from the centres R[0::2] (n_rep, 3N) and the modes (n_rep / 2, 3N); forces(R) -> (E
    (n_rep,), F).  Returns {'R', 'F', 'E' (whole handle, final positions), 'n_steps', 'converged', 'fmax',
    'curvature', 'n_rot', 'modes', 'phase', 'C_use' (the last translation's curvature, NaN before one), 'c2' (the last
    rotation's cos 2phi, NaN before one)}."""
    R = np.array(R, dtype=np.float64)
    nd, dimi = R.shape[0] // 2, R.shape[1]
    D = float(separation)
    c_t, s_t = float(cos_trial), float(sin_trial)
    s2_t, omc2_t = 2.0 * s_t * c_t, 2.0 * s_t * s_t
    N = np.array([init_mode(modes[d], R[2 * d], project_) for d in range(nd)]).reshape(nd, dimi)
    R[1::2] = R[0::2] + D * N
    T = np.zeros((nd, dimi))
    V = np.zeros((nd, dimi))
    fire = [_Fire() for _ in range(nd)]
    phase = np.zeros(nd, dtype=np.int64)
    C_N, C0, b1 = np.zeros(nd), np.zeros(nd), np.zeros(nd)
    n_rot = np.zeros(nd, dtype=np.int64)
    conv = np.zeros(nd, dtype=bool)
    f2 = np.zeros(nd)
    C_use, c2_last = np.full(nd, np.nan), np.full(nd, np.nan)
    thr = fmax * fmax

    def evaluate():
        E, F = forces(R)
        return np.asarray(E, dtype=np.float64).reshape(2 * nd), np.asarray(F, dtype=np.float64).reshape(R.shape)

    def test(F):
        for d in np.flatnonzero(~conv):
            f0, f1 = F[2 * d], F[2 * d + 1]
            if phase[d] == EVAL_N:
                C_N[d] = block_sum((f0 - f1) * N[d]) / D
            f2[d] = atom_max2(f0)
            conv[d] = f2[d] < thr and C_N[d] < 0.0

    def step(d, F):
        f0, f1, n = F[2 * d], F[2 * d + 1], N[d]
        if phase[d] == EVAL_N:
            G = (f1 - f0) / D
            g = block_sum(G * n)
            P = G - g * n
            f = math.sqrt(block_sum(P * P))
            if not (f < rot_min) and f != 0.0:
                T[d] = P / f
                R[2 * d + 1] = R[2 * d] + D * (c_t * n + s_t * T[d])
                C0[d], b1[d], phase[d] = C_N[d], -f, TRIAL
                return
            cu = C_N[d]
        else:
            nt = c_t * n + s_t * T[d]
            ct = block_sum((f0 - f1) * nt) / D
            a1 = ((C0[d] - ct) + b1[d] * s2_t) / omc2_t
            r = math.sqrt(a1 * a1 + b1[d] * b1[d])
            c2, s2 = (-a1) / r, (-b1[d]) / r
            if c2 >= 0.0:
                c = math.sqrt((1.0 + c2) / 2.0)
                s = s2 / (2.0 * c)
            else:
                s = math.sqrt((1.0 - c2) / 2.0)
                c = s2 / (2.0 * s)
            N[d], _ = project(c * n + s * T[d], R[2 * d], project_)
            n = N[d]
            cu = (C0[d] - a1) - r
            n_rot[d] += 1
            c2_last[d] = c2
        p = block_sum(f0 * n)
        Fd = f0 - (2.0 * p) * n if cu < 0.0 else -(p * n)
        fire[d].update(R[2 * d], V[d], Fd, dt, dtmax, maxstep)
        R[2 * d + 1] = R[2 * d] + D * n
        phase[d] = EVAL_N
        C_use[d] = cu

    E, F = evaluate()
    for _ in range(max_steps):
        test(F)
        if conv.all():
            break
        for d in np.flatnonzero(~conv):
            step(d, F)
        E, F = evaluate()
    test(F)
    return {'R': R, 'F': F, 'E': E, 'n_steps': np.array([z.n_steps for z in fire], dtype=np.int64),
            'converged': conv.copy(), 'fmax': np.sqrt(f2), 'curvature': C_N.copy(), 'n_rot': n_rot, 'modes': N,
            'phase': phase, 'C_use': C_use, 'c2': c2_last}
