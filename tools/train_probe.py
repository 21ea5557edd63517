"""Times GDMLTrain.train on a synthetic workload and prints the per-kernel-family device times.
usage: python tools/train_probe.py aspirin 250 [--profile] [--variant V]"""
import argparse, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import sgdml_b200
from sgdml_b200 import _lib, synth

ap = argparse.ArgumentParser()
ap.add_argument('workload'); ap.add_argument('n_train', type=int)
ap.add_argument('--profile', action='store_true'); ap.add_argument('--variant', type=int, default=3, choices=(0, 2, 3))
ap.add_argument('--reps', type=int, default=1)
a = ap.parse_args()
L = _lib.lib()
L.sgdml_b200_set_gemm_variant(a.variant)
cfg = dict(synth.CONFIGS[a.workload]); cfg['n_train'] = a.n_train
N, M = cfg['n_atoms'], cfg['n_train']
perms = synth.rotor_swap_group(N, cfg['n_rotors'], cfg['n_swaps'])
task = synth.make_task(N, M, perms, cfg['sig'])
tr = sgdml_b200.GDMLTrain()
tr.train(synth.make_task(N, 40, perms, cfg['sig']))
torch.cuda.synchronize()
for rep in range(a.reps):
    L.sgdml_b200_profile_reset(); L.sgdml_b200_profile_enable(1 if a.profile else 0)
    print('train start', N, M, flush=True)
    t0 = time.perf_counter(); model = tr.train(task); torch.cuda.synchronize(); dt = time.perf_counter() - t0
    L.sgdml_b200_profile_enable(0)
    n = 3 * N * M
    out = {'workload': a.workload, 'n_train': M, 'n': n, 'total_s': dt, 'timings': tr.timings, 'variant': a.variant,
           'solve_tflops': n ** 3 / 3 / tr.timings['solve_s'] * 1e-12, 'profiled': a.profile,
           'families_ms_scopes_launches': _lib.profile_snapshot()}
    print(json.dumps(out), flush=True)
