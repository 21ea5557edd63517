"""Dimer-steps per second of GDMLDimer on the device against the host loop it replaces.

A dimer step is one force evaluation of a dimer's centre and image; a rotating iteration takes two (the mode's, then
the trial's), a translating-only one takes one.  For the ethanol and aspirin synthetic models (synth.random_model on
the benchmark's shapes), dimers from random geometries with random modes, n_dimers = 1, 16 and 512:
  device: GDMLDimer.search with fmax = 0 (every dimer takes every step) and rot_min = 0 (every iteration rotates);
          wall clock around calls that end in a device synchronise, after a warm-up call
  host:   one GDMLPredict.predict of every centre and image per dimer step plus a NumPy dimer step (rotation by the
          same curvature fit, FIRE translation), written with np.einsum sums rather than the bit-exact restatement of
          tests/dimer_oracle.py, whose emulated summation tree is several times slower; the rigid projection is left
          out of the host loop, which flatters it slightly
Each rate is the median of `--reps` timed windows of about `--window` seconds.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
from relax_probe import _gpu_info, _rate  # noqa: E402

_D = 1e-4
_CT = _ST = math.sqrt(0.5)


def _dot(a, b):
    return np.einsum('bi,bi->b', a, b)


def _host_dimer(gp, R0, N0, n, dt, dtmax, maxstep=0.1):
    """n dimer steps of every dimer (centres R0, unit modes N0, (nd, 3N)) with one predict of all pairs per step."""
    nd, dimi = R0.shape
    R, N = R0.copy(), N0.copy()
    V = np.zeros_like(R)
    dts = np.full(nd, dt)
    a = np.full(nd, 0.1)
    n_pos = np.zeros(nd, dtype=int)
    first = True
    for s in range(n // 2):
        _, F = gp.predict(np.stack([R, R + _D * N], 1).reshape(2 * nd, dimi))
        F = F.reshape(nd, 2, dimi)
        f0, f1 = F[:, 0], F[:, 1]
        G = (f1 - f0) / _D
        P = G - _dot(G, N)[:, None] * N
        f = np.sqrt(_dot(P, P))
        T = P / np.where(f == 0.0, 1.0, f)[:, None]
        C0 = _dot(f0 - f1, N) / _D
        Nt = _CT * N + _ST * T
        _, F = gp.predict(np.stack([R, R + _D * Nt], 1).reshape(2 * nd, dimi))
        f1 = F.reshape(nd, 2, dimi)[:, 1]
        Ct = _dot(f0 - f1, Nt) / _D
        b1 = -f
        a1 = (C0 - Ct + b1 * 2.0 * _ST * _CT) / (2.0 * _ST * _ST)
        phi = 0.5 * np.arctan2(-b1, -a1)
        N = np.cos(phi)[:, None] * N + np.sin(phi)[:, None] * T
        N /= np.maximum(np.sqrt(_dot(N, N)), 1e-300)[:, None]
        cu = C0 - a1 - np.sqrt(a1 * a1 + b1 * b1)
        p = _dot(f0, N)
        Fd = np.where((cu < 0.0)[:, None], f0 - 2.0 * p[:, None] * N, -p[:, None] * N)
        if not first:
            Pw = _dot(Fd, V)
            up = Pw > 0.0
            c = np.where(up, a * np.sqrt(_dot(V, V)) / np.maximum(np.sqrt(_dot(Fd, Fd)), 1e-300), 0.0)
            V = np.where(up[:, None], (1.0 - a)[:, None] * V + c[:, None] * Fd, 0.0)
            grow = up & (n_pos > 5)
            dts = np.where(grow, np.minimum(dts * 1.1, dtmax), np.where(up, dts, dts * 0.5))
            a = np.where(grow, a * 0.99, np.where(up, a, 0.1))
            n_pos = np.where(up, n_pos + 1, 0)
        first = False
        V = V + dts[:, None] * Fd
        dr = dts[:, None] * V
        dr *= np.minimum(1.0, maxstep / np.maximum(np.sqrt(_dot(dr, dr)), 1e-300))[:, None]
        R += dr
    return R


def _workload(name, dimer_counts, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'rows': []}
    nd_max = max(dimer_counts)
    X = synth.geometries(N, nd_max, 1, r0=r0).reshape(nd_max, N, 3)
    modes = np.random.default_rng(0).standard_normal((nd_max, N, 3))
    for nd in dimer_counts:
        dim = sgdml_b200.GDMLDimer(gp, nd)
        conv = 1.0 / dim.F_to_eV_Ang  # eV -> the model's kcal/mol, as 1 / F_to_eV_Ang with Angstrom lengths

        def dev(n):
            dim.search(X[:nd], modes[:nd], fmax=0.0, max_steps=n, rot_min=0.0)
            torch.cuda.synchronize()

        dev(20)  # capture and warm-up
        sps, n = _rate(dev, window, reps)
        R0 = X[:nd].reshape(nd, 3 * N)
        N0 = modes[:nd].reshape(nd, 3 * N)
        N0 = N0 / np.linalg.norm(N0, axis=1, keepdims=True)

        def host(n):
            _host_dimer(gp, R0, N0, n, 0.1 / np.sqrt(conv), 1.0 / np.sqrt(conv))

        host(4)
        hsps, _ = _rate(host, window, reps)
        row = {'n_dimers': nd, 'device_dimer_steps_per_s': sps * nd, 'host_dimer_steps_per_s': hsps * nd,
               'speedup': sps / hsps, 'device_steps_per_window': n}
        print(json.dumps(row), flush=True)
        res['rows'].append(row)
        del dim
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
