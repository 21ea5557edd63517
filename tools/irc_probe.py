"""IRC points per second of GDMLIRC on the device against the host loop it replaces.

An IRC point is one RK4 step of one branch: four force evaluations.  For the ethanol and aspirin synthetic models
(synth.random_model on the benchmark's shapes), n_saddles = 1, 16 and 256 random geometries with random modes, two
branches each:
  device: GDMLIRC.run with fmax = 0, relax_ends = False and a step small enough that a descending branch runs to
          max_points, so every call replays 4 (max_points - 1) times; frozen branches (a branch whose first point
          rises) are still evaluated with the batch and count as the points they pay for.  Wall clock around calls
          that end in a device synchronise, after a warm-up call.
  host:   per RK4 stage one GDMLPredict.predict of every branch plus the NumPy stage in mass-weighted coordinates
          (np.einsum norms, not the bit-exact restatement of tests/irc_oracle.py).
Each rate is the median of `--reps` timed windows of about `--window` seconds.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
from relax_probe import _gpu_info, _rate  # noqa: E402

_STEP = 1e-4  # amu^1/2 Angstrom


def _host_irc(gp, R, r, n, h):
    """n RK4 points of every branch (R (n_rep, 3N) model units, r (3N,) sqrt of the inverse masses)."""
    def d(R):
        _, F = gp.predict(R)
        g = r * F
        return g / np.maximum(np.sqrt(np.einsum('bi,bi->b', g, g)), 1e-300)[:, None]

    for _ in range(n):
        k1 = d(R)
        k2 = d(R + r * (0.5 * h * k1))
        k3 = d(R + r * (0.5 * h * k2))
        k4 = d(R + r * (h * k3))
        R = R + r * ((h / 6.0) * (k1 + 2.0 * k2 + 2.0 * k3 + k4))
    return R


def _workload(name, counts, window, reps):
    import math

    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    masses = 1.0 + 15.0 * np.random.default_rng(3).random(N)
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'rows': []}
    n_max = max(counts)
    X = synth.geometries(N, n_max, 1, r0=r0).reshape(n_max, N, 3)
    modes = np.random.default_rng(0).standard_normal((n_max, N, 3))
    for ns in counts:
        irc = sgdml_b200.GDMLIRC(gp, masses, ns)

        def dev(n):
            irc.run(X[:ns], modes[:ns], step=_STEP, max_points=n + 1, fmax=0.0, relax_ends=False)
            torch.cuda.synchronize()

        dev(5)  # capture and warm-up
        pps, n = _rate(dev, window, reps)
        r = np.sqrt(np.repeat(irc.inv_mass, 3))
        h = _STEP * irc.Ang_to_R / math.sqrt(irc.F_to_eV_Ang * irc.Ang_to_R * sgdml_b200.md.FS ** 2)
        R = np.repeat(X[:ns].reshape(ns, 3 * N) * irc.Ang_to_R, 2, axis=0)

        def host(n):
            _host_irc(gp, R, r, n, h)

        host(2)
        hpps, _ = _rate(host, window, reps)
        row = {'n_saddles': ns, 'device_branch_points_per_s': pps * 2 * ns, 'host_branch_points_per_s': hpps * 2 * ns,
               'speedup': pps / hpps, 'device_points_per_window': n}
        print(json.dumps(row), flush=True)
        res['rows'].append(row)
        del irc
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
        res[name] = _workload(name, (1, 16, 256), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
