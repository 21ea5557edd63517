"""Replica-steps per second of GDMLReplicaExchange on the device against plain GDMLDynamics at the same replica count.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes), ladders of 8 and 16
temperatures (geometric, 300 to 600 K), 1 and 64 ladders:
  remd: the engine's sgdml_b200_remd_run through GDMLReplicaExchange.run, friction 0.01 / fs, exchange_every = 1 and
        100, no frames
  md:   GDMLDynamics.run with the same replica count at 300 K and the same friction (one step graph of k_md_step and the
        forces, no exchange kernel)
Wall clock around runs that end in a device synchronise, after a warm-up run; each rate is the median of `--reps`
timed windows of about `--window` seconds.  The exchange kernel's own time per step is not separated out: the
difference between the two rates includes it and the extra launch per step.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
from md_probe import _gpu_info, _rate  # noqa: E402


def _workload(name, ladders, n_temps_list, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    masses = np.full(N, 12.0)
    dt, fric = 0.5, 0.01
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'dt_fs': dt, 'rows': []}
    Rall = synth.geometries(N, max(ladders) * max(n_temps_list), 1, r0=r0)
    for n_temps in n_temps_list:
        T = np.geomspace(300.0, 600.0, n_temps)
        for n_l in ladders:
            B = n_l * n_temps
            row = {'n_temps': n_temps, 'n_ladders': n_l, 'B': B}
            rex = sgdml_b200.GDMLReplicaExchange(gp, masses, T, n_ladders=n_l)
            dyn = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=B)
            runs = {'md': lambda n: dyn.run(n, dt, temperature_K=300.0, friction_per_fs=fric)}
            for every in (1, 100):
                runs['remd_every_%d' % every] = lambda n, e=every: rex.run(n, dt, fric, e)
            rex.set_state(Rall[:B].reshape(n_l, n_temps, N, 3))
            dyn.set_state(Rall[:B])
            for label, fn in runs.items():
                def step(n, fn=fn):
                    fn(n)
                    torch.cuda.synchronize()

                step(20)  # capture and warm-up
                sps, n = _rate(step, window, reps)
                row[label + '_replica_steps_per_s'] = sps * B
                row[label + '_steps_per_window'] = n
            row['remd_every_1_over_md'] = row['remd_every_1_replica_steps_per_s'] / row['md_replica_steps_per_s']
            row['remd_every_100_over_md'] = row['remd_every_100_replica_steps_per_s'] / row['md_replica_steps_per_s']
            print(json.dumps(row), flush=True)
            res['rows'].append(row)
            del rex, dyn
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
        res[name] = _workload(name, (1, 64), (8, 16), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
