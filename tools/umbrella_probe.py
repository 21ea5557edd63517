"""Replica-steps per second of GDMLUmbrellaSampling on the device against plain GDMLDynamics (md_run) at the same
replica count, the device time of k_umbrella_bias and k_umbrella_exchange, and the time of MBAR on the device against
the NumPy MBAR of tests/umbrella_oracle.py.

Dynamics: the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes), two CVs (the distance
0-1 and the dihedral 0-1-2-3), B = 16, 256 and 4096 replicas as B / 16 ladders of 16 windows, 300 K, friction 0.01 / fs,
no frames, exchanges every 10 steps and none.  Wall clock around runs that end in a device synchronise, after a warm-up
run; each rate is the median of `--reps` timed windows of about `--window` seconds.  The kernels' own times are the
mean device time of their launches in a separate torch.profiler run with CUDA activities.
MBAR: K = 32 windows along one CV (a distance) and along two (distance and dihedral), n = 10^5, 10^6 and 10^7 samples
drawn from the biased Gaussians, tol 1e-10.  Time to convergence (one call, after a warm-up call at the smallest size)
and per iteration; the NumPy MBAR to convergence up to `--numpy-max` samples, and its time per iteration (five
iterations) up to `--numpy-iter-max`.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
from md_probe import _gpu_info, _rate  # noqa: E402

CVS = [('distance', (0, 1)), ('dihedral', (0, 1, 2, 3))]
NW = 16


def _kernel_us(fn, names):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for name in names:
        t = [e.device_time_total for e in prof.events() if name in e.name]
        out[name + '_us'] = float(np.mean(t)) if t else None
    return out


def _dynamics(name, batches, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    gp = sgdml_b200.GDMLPredict(synth.random_model(N, M, perms, cfg['sig'], r0=r0))
    masses = np.full(N, 12.0)
    dt, fric, T = 0.5, 0.01, 300.0
    res = {'workload': name, 'N': N, 'M': M, 'dt_fs': dt, 'n_cv': len(CVS), 'windows': NW, 'rows': []}
    Rall = synth.geometries(N, max(batches), 1, r0=r0)
    for B in batches:
        md = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=B)
        md.set_state(Rall[:B])

        def md_step(n):
            md.run(n, dt, temperature_K=T, friction_per_fs=fric)
            torch.cuda.synchronize()

        md_step(20)
        md_sps, _ = _rate(md_step, window, reps)
        probe = sgdml_b200.GDMLUmbrellaSampling(gp, masses, CVS, np.ones((NW, 2)), np.zeros((NW, 2)))
        probe.set_state(Rall[:1].reshape(1, N, 3))
        s0 = probe.get_state()['cv'][0, 0]
        del probe
        centers = s0 + np.stack([np.linspace(-0.1, 0.1, NW), np.linspace(-0.3, 0.3, NW)], 1)
        centers[:, 1] = (centers[:, 1] + np.pi) % (2 * np.pi) - np.pi
        us = sgdml_b200.GDMLUmbrellaSampling(gp, masses, CVS, centers, np.tile([5.0, 0.5], (NW, 1)),
                                             n_ladders=B // NW)
        us.set_state(Rall[:B].reshape(B // NW, NW, N, 3))
        for every in (10, 0):
            def us_step(n):
                us.run(n, dt, T, fric, exchange_every=every)
                torch.cuda.synchronize()

            us_step(20)
            sps, n = _rate(us_step, window, reps)
            row = {'B': B, 'exchange_every': every, 'umbrella_replica_steps_per_s': sps * B,
                   'md_replica_steps_per_s': md_sps * B, 'umbrella_over_md': sps / md_sps, 'steps_per_window': n}
            row.update(_kernel_us(lambda: us_step(20), ('k_umbrella_bias', 'k_umbrella_exchange')))
            print(json.dumps(row), flush=True)
            res['rows'].append(row)
        del md, us
    return res


def _mbar(sizes, numpy_max, numpy_iter_max):
    import torch

    import sgdml_b200
    import umbrella_oracle
    from sgdml_b200 import synth

    K, beta = 32, 1.0
    cfg = synth.CONFIGS['ethanol']  # MBAR reads only the CVs; the handle supplies the CV definitions
    perms, r0 = synth.config_perms_and_r0('ethanol')
    gp = sgdml_b200.GDMLPredict(synth.random_model(cfg['n_atoms'], cfg['n_train'], perms, cfg['sig'], r0=r0))
    rows = []
    for n_cv in (1, 2):
        cvs = CVS[:n_cv]
        centers = np.stack([np.linspace(1.0, 2.0, K), np.linspace(-2.5, 2.5, K)], 1)[:, :n_cv]
        kappas = np.tile([1000.0, 40.0], (K, 1))[:, :n_cv]
        us = sgdml_b200.GDMLUmbrellaSampling(gp, np.full(gp.n_atoms, 12.0), cvs, centers, kappas, E_to_eV=1.0,
                                             F_to_eV_Ang=1.0)
        rng = np.random.default_rng(0)
        for n in sizes:
            nk = n // K
            S = np.concatenate([c + rng.standard_normal((nk, n_cv)) / np.sqrt(beta * kappas[0]) for c in centers])
            if n_cv == 2:
                S[:, 1] = (S[:, 1] + np.pi) % (2 * np.pi) - np.pi
            Sd = torch.from_numpy(S).cuda()
            us._mbar_raw(Sd[:K * 1000], [1000] * K, beta, centers, kappas)  # warm-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f, _, it, resid = us._mbar_raw(Sd, [nk] * K, beta, centers, kappas, 1e-10, 100000)
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            row = {'K': K, 'n_cv': n_cv, 'n': K * nk, 'device_s': t, 'device_iterations': it,
                   'device_ms_per_iteration': 1e3 * t / it, 'resid': resid}
            if K * nk <= numpy_iter_max:
                u = np.array([beta * umbrella_oracle.restraint(S, [k for k, _ in cvs], centers[k2], kappas[k2])[0]
                              for k2 in range(K)])
                full = K * nk <= numpy_max  # to convergence, else 5 iterations for the time per iteration
                t0 = time.perf_counter()
                fn, _, itn = umbrella_oracle.mbar(u, [nk] * K, 1e-10, 100000 if full else 5)
                tn = time.perf_counter() - t0
                row.update(numpy_iterations=itn, numpy_ms_per_iteration=1e3 * tn / itn)
                if full:
                    row.update(numpy_s=tn, max_abs_df=float(np.max(np.abs(f.cpu().numpy() - fn))))
            print(json.dumps(row), flush=True)
            rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--window', type=float, default=0.3, help='seconds per timed window')
    ap.add_argument('--numpy-max', type=int, default=100000, help='largest pool the NumPy MBAR runs to convergence')
    ap.add_argument('--numpy-iter-max', type=int, default=1000000,
                    help='largest pool the NumPy MBAR runs five iterations on (the time per iteration)')
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    from sgdml_b200 import _lib

    _lib.require_gpu()
    res = {'gpu': _gpu_info()}
    print(json.dumps(res), flush=True)
    for name in ('ethanol', 'aspirin'):
        res[name] = _dynamics(name, (16, 256, 4096), a.window, a.reps)
    res['mbar'] = _mbar((100000, 1000000, 10000000), a.numpy_max, a.numpy_iter_max)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
