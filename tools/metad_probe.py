"""Replica-steps per second of GDMLMetadynamics on the device against plain GDMLDynamics (md_run) at the same replica
count, and the time of k_metad_bias itself.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes), with two CVs (the distance
0-1 and the dihedral 0-1-2-3), B = 1, 16, 256 and 4096 walkers in one group, and 0, 10^3 and 10^4 committed hills
(random centres, set with set_hills before the timed runs):
  metad: GDMLMetadynamics.run, 300 K, friction 0.01 / fs, no frames, a pace longer than the run (so the timed windows
         add no hills and every step sums the same hills): one step graph of k_md_step, the forces and k_metad_bias
  md:    GDMLDynamics.run with the same replica count, temperature and friction
The cost model is O(hills n_cv) per replica per step.  Wall clock around runs that end in a device synchronise, after a
warm-up run; each rate is the median of `--reps` timed windows of about `--window` seconds.  k_metad_bias's own time is
the mean device time of its launches in a separate torch.profiler run with CUDA activities (the profiler makes the
driver launch the step's kernels one by one).  Prints JSON with the card's name, power limit and max SM clock read in
the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
from md_probe import _gpu_info, _rate  # noqa: E402

CVS = [('distance', (0, 1)), ('dihedral', (0, 1, 2, 3))]


def _bias_kernel_us(fn):
    """mean device time (us) of the k_metad_bias launches of fn(), from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    times = [e.device_time_total for e in prof.events() if 'k_metad_bias' in e.name]
    return float(np.mean(times)) if times else None


def _workload(name, batches, hill_counts, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    gp = sgdml_b200.GDMLPredict(model)
    masses = np.full(N, 12.0)
    dt, fric, T = 0.5, 0.01, 300.0
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'dt_fs': dt, 'n_cv': len(CVS), 'rows': []}
    Rall = synth.geometries(N, max(batches), 1, r0=r0)
    rng = np.random.default_rng(0)
    for B in batches:
        md = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=B)
        md.set_state(Rall[:B])

        def md_step(n):
            md.run(n, dt, temperature_K=T, friction_per_fs=fric)
            torch.cuda.synchronize()

        md_step(20)
        md_sps, _ = _rate(md_step, window, reps)
        mt = sgdml_b200.GDMLMetadynamics(gp, masses, CVS, n_walkers=B)
        mt.set_state(Rall[:B].reshape(1, B, N, 3))
        s0 = mt.get_state()['cv'].reshape(B, -1)
        for H in hill_counts:
            c = s0[rng.integers(0, B, H)] + rng.normal(0.0, 0.1, (H, len(CVS)))
            mt.set_hills([{'centers': c, 'widths': np.full((H, len(CVS)), 0.1), 'heights': np.full(H, 1e-3)}])

            def mt_step(n):
                mt.run(n, dt, T, fric, 1e-3, [0.1, 0.1], 1 << 40, bias_factor=10.0)
                torch.cuda.synchronize()

            mt_step(20)  # capture and warm-up
            sps, n = _rate(mt_step, window, reps)
            row = {'B': B, 'hills': H, 'metad_replica_steps_per_s': sps * B, 'md_replica_steps_per_s': md_sps * B,
                   'metad_over_md': sps / md_sps, 'metad_steps_per_window': n,
                   'k_metad_bias_us': _bias_kernel_us(lambda: mt_step(20))}
            print(json.dumps(row), flush=True)
            res['rows'].append(row)
        del md, mt
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
        res[name] = _workload(name, (1, 16, 256, 4096), (0, 1000, 10000), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
