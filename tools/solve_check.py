#!/usr/bin/env python
"""Independent check of a trained model: the K.v identity (iterative.py:183-204) evaluates
(K - lam I) alphas with the PREDICTOR kernels, which share no code with the assembly and Cholesky
kernels that produced alphas, and compares it with the labels y (analytic.py:65-99 solves exactly this
system).  Also reports the force error on a sample of training points.

    python tools/solve_check.py --workload aspirin --n-train 300        # n = 18900 (NBO = 1024 path)
    SGDML_B200_OZAKI_SLICES=7 python tools/solve_check.py ...          # int8 (wgmma) trailing updates
"""

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


from sgdml_b200.diagnostics import residual_report  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='aspirin')
    ap.add_argument('--n-train', type=int, default=None)
    ap.add_argument('--repeat', type=int, default=1, help='timed training runs (the first one allocates the workspaces)')
    ap.add_argument('--profile', action='store_true', help='per-kernel-family device times (adds synchronisation)')
    args = ap.parse_args()
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    task = synth.make_config_task(args.workload, n_train=args.n_train)
    M, N = task['R_train'].shape[:2]
    tr = sgdml_b200.GDMLTrain()
    tr.train(synth.make_config_task(args.workload, n_train=min(M, 40)))  # warm-up
    from sgdml_b200 import _lib

    for it in range(args.repeat):
        if args.profile:
            _lib.lib().sgdml_b200_profile_reset()
            _lib.lib().sgdml_b200_profile_enable(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model = tr.train(task)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if args.profile:
            _lib.lib().sgdml_b200_profile_enable(0)
            print('profile (ms, scopes, launches):', {k: (round(v[0], 1), v[1], v[2]) for k, v in _lib.profile_snapshot().items()}, file=sys.stderr)
        rep = residual_report(model, task)
        rep.update({'workload': args.workload, 'n': 3 * N * M, 'train_s': dt, 'timings': tr.timings, 'run': it,
                    'ozaki_slices': os.environ.get('SGDML_B200_OZAKI_SLICES', 'default')})
        print(json.dumps(rep), flush=True)


if __name__ == '__main__':
    main()
