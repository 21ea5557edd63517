"""NumPy restatement of the device nudged elastic band (csrc/md.cu k_neb_force / k_neb_fire_step, sgdml_b200_neb_fire):
the NEB force of every interior image in the kernel's order and roundings (md.cuh), and FIRE on each band's interior
images as one vector, which is relax_oracle.fire driven by the NEB forces.

Replica b P + j of an (n_rep, 3N) array is image j of band b; images 0 and P - 1 are fixed.  NumPy never fuses a
multiply and an add, so with the same model forces the results agree with the kernels bit for bit.
"""

import numpy as np

import relax_oracle
from relax_oracle import block_sum


def climbing_index(E):
    """The highest interior image of every band, the lowest index on ties: E (n_bands, P) -> (n_bands,) int."""
    E = np.asarray(E, dtype=np.float64)
    top = np.ones(E.shape[0], dtype=np.int64)
    for j in range(2, E.shape[1] - 1):
        top = np.where(E[:, j] > E[np.arange(E.shape[0]), top], j, top)
    return top


def neb_force(R, F, E, P, k, climb):
    """k_neb_force: R, F (n_rep, 3N) and E (n_rep,) of the model -> (F_neb (n_bands, (P - 2) 3N) of the interior
    images, the climbing index (n_bands,))."""
    R = np.asarray(R, dtype=np.float64)
    dimi = R.shape[-1]
    R = R.reshape(-1, P, dimi)
    F = np.asarray(F, dtype=np.float64).reshape(-1, P, dimi)
    E = np.asarray(E, dtype=np.float64).reshape(-1, P)
    top = climbing_index(E)
    out = np.empty((R.shape[0], P - 2, dimi))
    for i in range(1, P - 1):
        e, ep, em = E[:, i], E[:, i + 1], E[:, i - 1]
        tp = R[:, i + 1] - R[:, i]
        tm = R[:, i] - R[:, i - 1]
        up = (ep > e) & (e > em)
        down = (ep < e) & (e < em)
        dp, dm = np.abs(ep - e), np.abs(em - e)
        dmax, dmin = np.where(dp > dm, dp, dm), np.where(dp > dm, dm, dp)
        wp, wm = np.where(ep > em, dmax, dmin), np.where(ep > em, dmin, dmax)
        tau = np.where(up[:, None], tp, np.where(down[:, None], tm, tp * wp[:, None] + tm * wm[:, None]))
        nt = np.sqrt(block_sum(tau * tau))
        n_p = np.sqrt(block_sum(tp * tp))
        n_m = np.sqrt(block_sum(tm * tm))
        with np.errstate(divide='ignore', invalid='ignore'):
            th = np.where((nt == 0.0)[:, None], 0.0, tau / nt[:, None])
        f = F[:, i]
        fd = block_sum(f * th)
        spring = k * (n_p - n_m)
        climbing = bool(climb) & (top == i)
        out[:, i - 1] = np.where(climbing[:, None], f - (2.0 * fd)[:, None] * th,
                                 (f - fd[:, None] * th) + spring[:, None] * th)
    return out.reshape(R.shape[0], (P - 2) * dimi), top


def neb_fire(forces, R, P, max_steps, fmax, k, climb, maxstep, dt, dtmax):
    """sgdml_b200_neb_fire from R (n_bands P, 3N); forces(R) -> (E (n_rep,), F) of the model.  Returns relax_oracle.fire's
    dict per band ('n_steps', 'converged', 'fmax' of the NEB forces, 'tested', ...) with 'R', 'F', 'E' replaced by the
    whole bands' positions, model forces and energies (n_rep, 3N) / (n_rep,) at the final positions, and 'climbing'
    (n_bands,) the highest interior image there."""
    R = np.array(R, dtype=np.float64)
    dimi = R.shape[1]
    nb = R.shape[0] // P
    ends = R.reshape(nb, P, dimi)[:, [0, P - 1]].copy()
    last = {}

    def band_forces(X):
        full = np.empty((nb, P, dimi))
        full[:, [0, P - 1]] = ends
        full[:, 1:P - 1] = X.reshape(nb, P - 2, dimi)
        full = full.reshape(nb * P, dimi)
        E, F = forces(full)
        E = np.asarray(E, dtype=np.float64).reshape(nb * P)
        F = np.asarray(F, dtype=np.float64).reshape(nb * P, dimi)
        Fn, top = neb_force(full, F, E, P, k, climb)
        last.update(R=full, F=F, E=E, climbing=top)
        return E.reshape(nb, P).max(1), Fn

    X0 = R.reshape(nb, P, dimi)[:, 1:P - 1].reshape(nb, (P - 2) * dimi)
    out = relax_oracle.fire(band_forces, X0, max_steps, fmax, maxstep, dt, dtmax)
    out.update(last)
    return out
