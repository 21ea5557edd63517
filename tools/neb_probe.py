"""Band-steps per second of GDMLNEB on the device against the host loop it replaces.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes), bands of 8 images between
two random geometries, n_bands = 1, 16 and 512:
  device: GDMLNEB.neb with fmax = 0 and climb on (every band takes every step); wall clock around calls that end in a
          device synchronise, after a warm-up call
  host:   one GDMLPredict.predict of every image of every band per step plus a NumPy NEB force and band FIRE step (the
          route of ASE's NEB on a calculator that evaluates the whole band at once), written with np.einsum sums rather
          than the bit-exact restatement of tests/neb_oracle.py, whose emulated summation tree is several times slower
Each rate is the median of `--reps` timed windows of about `--window` seconds.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
from relax_probe import _gpu_info, _rate  # noqa: E402

P = 8


def _host_neb_force(R, F, E, k, climb):
    """NEB forces (nb, P - 2, 3N) of bands R, F (nb, P, 3N), E (nb, P): the improved tangent, spring, climbing image."""
    tp, tm = R[:, 2:] - R[:, 1:-1], R[:, 1:-1] - R[:, :-2]
    e, ep, em = E[:, 1:-1], E[:, 2:], E[:, :-2]
    dp, dm = np.abs(ep - e), np.abs(em - e)
    dmax, dmin = np.maximum(dp, dm), np.minimum(dp, dm)
    wp = np.where(ep > em, dmax, dmin)
    wm = np.where(ep > em, dmin, dmax)
    tau = np.where(((ep > e) & (e > em))[..., None], tp,
                   np.where(((ep < e) & (e < em))[..., None], tm, tp * wp[..., None] + tm * wm[..., None]))
    nt = np.sqrt(np.einsum('bij,bij->bi', tau, tau))
    th = tau / np.where(nt == 0.0, 1.0, nt)[..., None]
    f = F[:, 1:-1]
    fd = np.einsum('bij,bij->bi', f, th)
    spring = k * (np.sqrt(np.einsum('bij,bij->bi', tp, tp)) - np.sqrt(np.einsum('bij,bij->bi', tm, tm)))
    out = f - fd[..., None] * th + spring[..., None] * th
    if climb:
        top = np.argmax(e, axis=1)
        b = np.arange(len(R))
        out[b, top] = f[b, top] - 2.0 * fd[b, top][:, None] * th[b, top]
    return out


def _host_neb(gp, R, n, k, dt, dtmax, maxstep=0.2):
    """n steps of FIRE on every band of R (nb, P, 3N) with NEB forces, one predict of all images per step."""
    nb, _, dimi = R.shape
    R = R.copy()
    V = np.zeros((nb, (P - 2) * dimi))
    dt = np.full(nb, dt)
    a = np.full(nb, 0.1)
    n_pos = np.zeros(nb, dtype=int)
    for s in range(n + 1):
        E, F = gp.predict(R.reshape(nb * P, dimi))
        Fn = _host_neb_force(R, F.reshape(nb, P, dimi), E.reshape(nb, P), k, True).reshape(nb, -1)
        if s == n:
            break
        if s > 0:
            Pw = np.einsum('bi,bi->b', Fn, V)
            up = Pw > 0.0
            vn = np.sqrt(np.einsum('bi,bi->b', V, V))
            fn = np.sqrt(np.einsum('bi,bi->b', Fn, Fn))
            c = np.where(up, a * vn / np.where(up, fn, 1.0), 0.0)
            V = np.where(up[:, None], (1.0 - a)[:, None] * V + c[:, None] * Fn, 0.0)
            grow = up & (n_pos > 5)
            dt = np.where(grow, np.minimum(dt * 1.1, dtmax), np.where(up, dt, dt * 0.5))
            a = np.where(grow, a * 0.99, np.where(up, a, 0.1))
            n_pos = np.where(up, n_pos + 1, 0)
        V = V + dt[:, None] * Fn
        dr = dt[:, None] * V
        nrm = np.sqrt(np.einsum('bi,bi->b', dr, dr))
        dr *= np.minimum(1.0, maxstep / np.maximum(nrm, 1e-300))[:, None]
        R[:, 1:-1] += dr.reshape(nb, P - 2, dimi)
    return R


def _workload(name, band_counts, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'images': P, 'rows': []}
    nb_max = max(band_counts)
    ends = synth.geometries(N, 2 * nb_max, 1, r0=r0).reshape(2, nb_max, N, 3)
    F_conv = None
    for nb in band_counts:
        neb = sgdml_b200.GDMLNEB(gp, P, n_bands=nb)
        F_conv = 1.0 / neb.F_to_eV_Ang
        images = neb.interpolate(ends[0, :nb], ends[1, :nb], P, align=False)

        def dev(n):
            neb.neb(images, fmax=0.0, max_steps=n, climb=True)
            torch.cuda.synchronize()

        dev(20)  # capture and warm-up
        sps, n = _rate(dev, window, reps)
        R = images.reshape(nb, P, 3 * N)

        def host(n):
            _host_neb(gp, R, n, 0.1 * F_conv, 0.1 / np.sqrt(F_conv), 1.0 / np.sqrt(F_conv))

        host(3)
        hsps, _ = _rate(host, window, reps)
        row = {'n_bands': nb, 'device_band_steps_per_s': sps * nb, 'host_band_steps_per_s': hsps * nb,
               'speedup': sps / hsps, 'device_steps_per_window': n}
        print(json.dumps(row), flush=True)
        res['rows'].append(row)
        del neb
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--window', type=float, default=0.3, help='seconds per timed window')
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    from sgdml_b200 import _lib

    _lib.require_gpu()
    res = {'gpu': _gpu_info()}
    print(json.dumps(res), flush=True)
    for name in ('ethanol', 'aspirin'):
        res[name] = _workload(name, (1, 16, 512), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
