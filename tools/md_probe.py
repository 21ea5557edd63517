"""Steps per second of GDMLDynamics on the device against the host loop it replaces.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes):
  device: GDMLDynamics.run at B = 1, 16, 256 and 4096 replicas, NVE (velocity Verlet) and Langevin (300 K,
          0.01 / fs), no frames; wall clock around runs that end in a device synchronise, after a warm-up run
  host:   at B = 1 and 16, the ASE-shaped route: GDMLPredict.predict on NumPy positions plus a NumPy velocity-Verlet
          step per call
Each figure is the median of `--reps` timed windows of about `--window` seconds.  Prints JSON with the card's name,
power limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

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


def _workload(name, batches, host_batches, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    masses = np.full(N, 12.0)
    dt = 0.5
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'dt_fs': dt, 'device': [], 'host': []}
    Rall = synth.geometries(N, max(batches), 1, r0=r0)
    for B in batches:
        dyn = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=B)
        row = {'B': B}
        for label, kw in (('nve', {}), ('langevin', {'temperature_K': 300.0, 'friction_per_fs': 0.01})):
            dyn.set_state(Rall[:B])

            def run(n):
                dyn.run(n, dt, **kw)
                torch.cuda.synchronize()

            run(20)  # capture and warm-up
            sps, n = _rate(run, window, reps)
            row[label + '_steps_per_s'] = sps
            row[label + '_replica_steps_per_s'] = sps * B
            row[label + '_steps_per_window'] = n
        print(json.dumps(row), flush=True)
        res['device'].append(row)
        del dyn
    s = np.repeat(sgdml_b200.GDMLDynamics(gp, masses).inv_mass, 3)  # model units per fs^2 per force unit
    h = 0.5 * dt
    for B in host_batches:
        state = {'R': Rall[:B].reshape(B, -1).copy(), 'V': np.zeros((B, 3 * N))}
        state['F'] = gp.predict(state['R'])[1]

        def host(n):
            R, V, F = state['R'], state['V'], state['F']
            for _ in range(n):
                V = V + h * (F * s)
                R = R + dt * V
                E, F = gp.predict(R)
                V = V + h * (F * s)
            state.update(R=R, V=V, F=F)

        host(20)
        sps, n = _rate(host, window, reps)
        row = {'B': B, 'host_steps_per_s': sps, 'host_replica_steps_per_s': sps * B, 'steps_per_window': n}
        print(json.dumps(row), flush=True)
        res['host'].append(row)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--window', type=float, default=0.5, help='seconds per timed window')
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    from sgdml_b200 import _lib

    _lib.require_gpu()
    res = {'gpu': _gpu_info()}
    print(json.dumps(res), flush=True)
    for name in ('ethanol', 'aspirin'):
        res[name] = _workload(name, (1, 16, 256, 4096), (1, 16), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
