"""Replica-steps per second of GDMLRelaxation on the device against the host loop it replaces, and the steps quenching
takes.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes):
  device: GDMLRelaxation.relax with fmax = 0 (every replica takes every step) at B = 1, 16, 256 and 4096, FIRE and
          L-BFGS (memory 20), and GDMLDynamics NVE on the same replicas for comparison; wall clock around calls that
          end in a device synchronise, after a warm-up call
  host:   at B = 1 and 16, the ASE-shaped route: GDMLPredict.predict on NumPy positions plus a plain NumPy optimiser
          step written as ASE's (np.vdot / np.dot sums, FIRE vectorised over replicas, L-BFGS's two-loop per replica),
          not the bit-exact restatement of tests/relax_oracle.py, whose emulated summation tree is several times slower
  quench: 256 Langevin frames (300 K, 0.01 / fs, 200 steps of 0.5 fs apart) relaxed to fmax = 0.05 eV/Angstrom with
          each optimiser (ASE's defaults, at most 1000 steps): percentiles of the steps taken, the converged fraction
          and the wall time
Each rate is the median of `--reps` timed windows of about `--window` seconds.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def _gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], text=True
        ).strip()
    except Exception as e:  # noqa: BLE001
        return 'unknown (%s)' % e


def _rate(step_fn, window, reps):
    """Median steps/s of step_fn(n) (which takes n steps and returns after a synchronise) over `reps` windows."""
    t0 = time.perf_counter()
    step_fn(10)
    per = max((time.perf_counter() - t0) / 10, 1e-7)
    n = max(10, int(window / per))
    rates = []
    for _ in range(reps):
        t0 = time.perf_counter()
        step_fn(n)
        rates.append(n / (time.perf_counter() - t0))
    return float(np.median(rates)), n


def _host_fire(forces, R, n, dt, dtmax, maxstep=0.2):
    """n steps of ASE's FIRE (mass-free, default constants) on every replica of R (B, 3N), vectorised over replicas."""
    V = np.zeros_like(R)
    dt = np.full(len(R), dt)
    a = np.full(len(R), 0.1)
    n_pos = np.zeros(len(R), dtype=int)
    _, F = forces(R)
    for k in range(n):
        if k > 0:
            P = np.einsum('bi,bi->b', F, V)
            up = P > 0.0
            vn = np.sqrt(np.einsum('bi,bi->b', V, V))
            fn = np.sqrt(np.einsum('bi,bi->b', F, F))
            c = np.where(up, a * vn / np.where(up, fn, 1.0), 0.0)
            V = np.where(up[:, None], (1.0 - a)[:, None] * V + c[:, None] * F, 0.0)
            grow = up & (n_pos > 5)
            dt = np.where(grow, np.minimum(dt * 1.1, dtmax), np.where(up, dt, dt * 0.5))
            a = np.where(grow, a * 0.99, np.where(up, a, 0.1))
            n_pos = np.where(up, n_pos + 1, 0)
        V = V + dt[:, None] * F
        dr = dt[:, None] * V
        nrm = np.sqrt(np.einsum('bi,bi->b', dr, dr))
        dr *= np.minimum(1.0, maxstep / np.maximum(nrm, 1e-300))[:, None]
        R = R + dr
        _, F = forces(R)
    return R


def _host_lbfgs(forces, R, n, h0, memory=20, maxstep=0.2):
    """n steps of L-BFGS on every replica of R (B, 3N): ASE's two-loop with np.dot, one history per replica."""
    B = len(R)
    hist = [[] for _ in range(B)]
    E, F = forces(R)
    r_prev = g_prev = E_prev = None
    for k in range(n):
        g = -F
        D = np.empty_like(R)
        for b in range(B):
            h = hist[b]
            if k > 0:
                s, y = R[b] - r_prev[b], g[b] - g_prev[b]
                sy = np.dot(s, y)
                if sy > 0.0 and E[b] <= E_prev[b]:
                    h.append((s, y, 1.0 / sy))
                    del h[:-memory]
                else:
                    h.clear()
            q = g[b].copy()
            al = []
            for s, y, rho in reversed(h):
                al.append(rho * np.dot(s, q))
                q -= al[-1] * y
            z = (np.dot(h[-1][0], h[-1][1]) / np.dot(h[-1][1], h[-1][1]) if h else h0) * q
            for (s, y, rho), ai in zip(h, reversed(al)):
                z += s * (ai - rho * np.dot(y, z))
            d = -z
            if np.dot(d, g[b]) >= 0.0:
                h.clear()
                d = -h0 * g[b]
            L = np.sqrt((d.reshape(-1, 3) ** 2).sum(1).max())
            D[b] = d * (maxstep / L) if L > maxstep else d
        r_prev, g_prev, E_prev = R, g, E
        R = R + D
        E, F = forces(R)
    return R


OPTS = {'fire': {'optimizer': 'fire'}, 'lbfgs': {'optimizer': 'lbfgs', 'memory': 20}}


def _workload(name, batches, host_batches, window, reps, n_quench):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'device': [], 'host': [], 'quench': []}
    Rall = synth.geometries(N, max(batches + (n_quench,)), 1, r0=r0)
    for B in batches:
        rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=B)
        dyn = sgdml_b200.GDMLDynamics(gp, np.full(N, 12.0), n_replicas=B)
        row = {'B': B}
        for label, kw in OPTS.items():
            def run(n):
                rel.relax(Rall[:B], fmax=0.0, max_steps=n, **kw)
                torch.cuda.synchronize()

            run(20)  # capture and warm-up
            sps, n = _rate(run, window, reps)
            row[label + '_replica_steps_per_s'] = sps * B
            row[label + '_steps_per_window'] = n
        dyn.set_state(Rall[:B])

        def md(n):
            dyn.run(n, 0.5)
            torch.cuda.synchronize()

        md(20)
        row['md_nve_replica_steps_per_s'] = _rate(md, window, reps)[0] * B
        print(json.dumps(row), flush=True)
        res['device'].append(row)
        del rel, dyn
    F_conv = 1.0 / sgdml_b200.GDMLRelaxation(gp).F_to_eV_Ang  # eV/Angstrom -> model force unit (Ang_to_R = 1)
    for B in host_batches:
        row = {'B': B}
        for label in OPTS:
            R = Rall[:B].reshape(B, -1).copy()

            def host(n, label=label, R=R):
                forces = gp.predict
                if label == 'fire':
                    _host_fire(forces, R, n, 0.1 / np.sqrt(F_conv), 1.0 / np.sqrt(F_conv))
                else:
                    _host_lbfgs(forces, R, n, 1.0 / (70.0 * F_conv))

            host(10)
            sps, n = _rate(host, window, reps)
            row['host_' + label + '_replica_steps_per_s'] = sps * B
        print(json.dumps(row), flush=True)
        res['host'].append(row)
    # quench Langevin frames
    dyn = sgdml_b200.GDMLDynamics(gp, np.full(N, 12.0), n_replicas=n_quench)
    dyn.set_state(Rall[:n_quench])
    frames = dyn.run(200, 0.5, temperature_K=300.0, friction_per_fs=0.01, seed=1, stride=200)['positions'][0]
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=n_quench)
    for label, kw in OPTS.items():
        rel.relax(frames, fmax=0.05, max_steps=5, **kw)  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = rel.relax(frames, fmax=0.05, max_steps=1000, **kw)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        ns = out['n_steps']
        row = {'optimizer': label, 'B': n_quench, 'converged_fraction': float(np.mean(out['converged'])),
               'steps_p10_p50_p90_max': [int(np.percentile(ns, q)) for q in (10, 50, 90)] + [int(ns.max())],
               'steps_mean': float(ns.mean()), 'seconds': t}
        print(json.dumps(row), flush=True)
        res['quench'].append(row)
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
        res[name] = _workload(name, (1, 16, 256, 4096), (1, 16), a.window, a.reps, 256)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
