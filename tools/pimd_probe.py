"""Steps per second of GDMLPathIntegralDynamics on the device, against classical GDMLDynamics on the same number of
replicas and, for one polymer, the host loop it replaces.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes), P in {8, 32} beads and
n_poly in {1, 16, 128} polymers:
  pimd:      GDMLPathIntegralDynamics.run at 300 K, PILE-L (lambda = 1, centroid friction 0.01 / fs), no frames
  classical: GDMLDynamics.run on n_poly P replicas, Langevin at 300 K, 0.01 / fs, no frames
  host:      at n_poly = 1, GDMLPredict.predict on the P bead geometries (NumPy) plus the bit-exact NumPy restatement
             of the ring-polymer step (tests/pimd_oracle.py, without noise) per call; its Python-level loop over the
             P^2 (mode, bead) pairs dominates, so this understates a vectorised host step
Wall clock around runs that end in a device synchronise, after a warm-up run; each figure is the median of `--reps`
windows of about `--window` seconds.  Prints JSON with the card's name, power limit and max SM clock read in the same
run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

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


def _workload(name, beads, polymers, window, reps):
    import torch

    import pimd_oracle
    import sgdml_b200
    from sgdml_b200 import md, synth
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc  # the models' energy unit

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    gp = sgdml_b200.GDMLPredict(synth.random_model(N, M, perms, cfg['sig'], r0=r0))
    masses = np.full(N, 12.0)
    dt, T = 0.5, 300.0
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'dt_fs': dt, 'rows': []}
    Rall = synth.geometries(N, max(polymers), 1, r0=r0)
    for P in beads:
        for n_poly in polymers:
            B = n_poly * P
            row = {'P': P, 'n_poly': n_poly, 'replicas': B}
            dyn = sgdml_b200.GDMLPathIntegralDynamics(gp, masses, P, n_poly)
            dyn.set_state(Rall[:n_poly])

            def run(n):
                dyn.run(n, dt, T, centroid_friction_per_fs=0.01, pile_lambda=1.0)
                torch.cuda.synchronize()

            run(20)  # capture and warm-up
            sps, n = _rate(run, window, reps)
            row.update(pimd_steps_per_s=sps, pimd_bead_steps_per_s=sps * B, pimd_steps_per_window=n)
            del dyn
            cl = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=B)
            cl.set_state(np.repeat(Rall[:n_poly], P, 0))

            def run_c(n):
                cl.run(n, dt, temperature_K=T, friction_per_fs=0.01)
                torch.cuda.synchronize()

            run_c(20)
            sps_c, _ = _rate(run_c, window, reps)
            row.update(classical_steps_per_s=sps_c, classical_replica_steps_per_s=sps_c * B,
                       pimd_over_classical=sps / sps_c)
            del cl
            if n_poly == 1:
                s = np.repeat(sgdml_b200.GDMLDynamics(gp, masses).inv_mass, 3)
                t = pimd_oracle.constants(P, dt, md.KB_EV * T / kc, md.HBAR_EV_FS / kc, 0.0, 0.0, s)
                R = np.repeat(Rall[:1].reshape(1, 1, -1), P, 1)
                state = {'R': R, 'V': np.zeros_like(R)}
                state['F'] = gp.predict(R.reshape(P, -1))[1].reshape(R.shape)

                def host(n):
                    R, V, F = state['R'], state['V'], state['F']
                    for _ in range(n):
                        V = V + t['h'] * (F * s)
                        Q, U = pimd_oracle.to_modes(t["C"], R), pimd_oracle.to_modes(t["C"], V)
                        Q, U = pimd_oracle.free_ring(t, Q, U)
                        Q, U = pimd_oracle.free_ring(t, Q, U)
                        R, V = pimd_oracle.from_modes(t['C'], Q), pimd_oracle.from_modes(t['C'], U)
                        F = gp.predict(R.reshape(P, -1))[1].reshape(R.shape)
                        V = V + t['h'] * (F * s)
                    state.update(R=R, V=V, F=F)

                host(5)
                sps_h, _ = _rate(host, window, reps)
                row.update(host_steps_per_s=sps_h, host_bead_steps_per_s=sps_h * P)
            print(json.dumps(row), flush=True)
            res['rows'].append(row)
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
        res[name] = _workload(name, (8, 32), (1, 16, 128), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
