"""NumPy restatement of the device MD integrator (csrc/md.cu, sgdml_b200_md_run): Philox4x32-10, the Box-Muller
normals drawn from it, and the BAOAB step with its roundings, driven by any force function.

With the same forces, the B and A updates below round exactly as the device's (__dmul_rn / __dadd_rn; NumPy never
fuses a multiply and an add), so positions and velocities agree bit for bit as long as the forces do.
"""

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: (..., 4) uint32-valued integers, key: (2,) -> (..., 4) uint32 output words."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r > 0:
            k0 = (k0 + _W0) & 0xFFFFFFFF
            k1 = (k1 + _W1) & 0xFFFFFFFF
        p0 = _M0 * c[0]
        p1 = _M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
    return np.stack([x.astype(np.uint32) for x in c], axis=-1)


def _uniform53(hi, lo):
    u = (hi.astype(np.uint64) << np.uint64(32)) | lo.astype(np.uint64)
    return ((u >> np.uint64(11)).astype(np.float64) + 0.5) * 2.0**-53


def normals(seed, step, n_rep, dimi):
    """xi (n_rep, dimi): the noise of global step `step` for every replica and coordinate."""
    n_pairs = (dimi + 1) // 2
    j, rep = np.meshgrid(np.arange(n_pairs, dtype=np.uint64), np.arange(n_rep, dtype=np.uint64))
    ctr = np.stack([j, rep, np.full_like(j, step & 0xFFFFFFFF), np.full_like(j, step >> 32)], axis=-1)
    u = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    ua, ub = _uniform53(u[..., 0], u[..., 1]), _uniform53(u[..., 2], u[..., 3])
    rad = np.sqrt(-2.0 * np.log(ua))
    xi = np.empty((n_rep, 2 * n_pairs))
    xi[:, 0::2] = rad * np.cos(2.0 * np.pi * ub)
    xi[:, 1::2] = rad * np.sin(2.0 * np.pi * ub)
    return xi[:, :dimi]


def constants(dt, gamma, kT, s):
    """h, c1, sigma (per coordinate) as the engine computes them on the host."""
    h = 0.5 * dt
    c1 = np.exp(-gamma * dt)
    return h, c1, np.sqrt((1.0 - c1 * c1) * kT * np.asarray(s, dtype=np.float64))


def kinetic(V, s):
    return 0.5 * (V * V / s).sum(-1)


def run(forces, R, V, s, n_steps, dt, gamma=0.0, kT=0.0, seed=0, step0=0, stride=0, F=None, E=None):
    """BAOAB from (R, V) (n_rep, 3N) with s (3N,) inverse masses per coordinate.  forces(R) -> (E (n_rep,), F).
    Returns the final (R, V, F, E) and the frames {'R', 'V', 'E_pot', 'E_kin'} after every stride-th step."""
    R = np.array(R, dtype=np.float64)
    V = np.array(V, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    if F is None:
        E, F = forces(R)
    h, c1, sigma = constants(dt, gamma, kT, s)
    frames = {'R': [], 'V': [], 'E_pot': [], 'E_kin': []}
    for k in range(n_steps):
        V = V + h * (F * s)
        R = R + h * V
        if gamma > 0.0:
            V = c1 * V + sigma * normals(seed, step0 + k, R.shape[0], R.shape[1])
        R = R + h * V
        E, F = forces(R)
        V = V + h * (F * s)
        if stride and (k + 1) % stride == 0:
            for key, val in (('R', R), ('V', V), ('E_pot', E), ('E_kin', kinetic(V, s))):
                frames[key].append(np.array(val))
    return (R, V, F, E), {k: np.array(v) for k, v in frames.items()}
