"""Times the all-pairs matching of the permutation search (sgdml_b200_bipartite_match) at the shapes DESIGN.md quotes:

    python tools/perm_probe.py [--reps 5] [--oracle-pairs 60]

For each (N atoms, M geometries, S planted symmetries) it prints the host preparation time (pair distances and M
eigen-decompositions, one process), the device time of the all-pairs call between CUDA events on device-resident
inputs (median of --reps after a warm-up call), pairs per second, where the cost matrix lives, and the oracle's
single-process time per pair (SciPy's linear_sum_assignment, oracle/perm.py) on a sample of pairs on the same host.
The GPU's name, power limit and maximum SM clock are read in the same run.  Needs a CUDA device: there is nothing to
fall back to."""

import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = [(9, 200, 6), (21, 1000, 6), (60, 1000, 6), (370, 200, 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--oracle-pairs', type=int, default=60)
    args = ap.parse_args()
    import torch

    from oracle import perm as operm
    from sgdml_b200 import _lib, synth
    from sgdml_b200 import perm as eperm

    _lib.require_gpu()
    gpu = subprocess.check_output(
        ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], text=True).strip()
    print('GPU (name, power limit, max SM clock): %s' % gpu.splitlines()[0])
    L = _lib.lib()
    for N, M, S in SHAPES:
        group = synth.rotor_swap_group(N, 1, 1 if S == 6 else 0)
        assert group.shape[0] == S
        R, z, _ = synth.planted_symmetry_geometries(N, M, group, 1)
        t0 = time.perf_counter()
        adj, absv = eperm.prepare(R)
        t_prep = time.perf_counter() - t0
        d_adj, d_absv = torch.from_numpy(adj).cuda(), torch.from_numpy(absv).cuda()
        n_pairs = M * (M - 1) // 2
        d_cost = torch.zeros((M, M), dtype=torch.float64, device='cuda')
        d_has = torch.zeros(n_pairs, dtype=torch.uint8, device='cuda')

        def call():
            _lib.check(L.sgdml_b200_bipartite_match(d_adj.data_ptr(), d_absv.data_ptr(), z.ctypes.data, M, N, None, 0,
                                                    d_cost.data_ptr(), None, d_has.data_ptr(), _lib.current_stream()),
                       'bipartite_match')

        call()  # warm-up: module load, workspace
        ms = []
        for _ in range(max(args.reps, 5)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        dev_ms = float(np.median(ms))
        rng = np.random.default_rng(0)
        sample = [(int(i), int(j)) for i, j in zip(rng.integers(0, M // 2, args.oracle_pairs),
                                                   rng.integers(M // 2, M, args.oracle_pairs))]
        t0 = time.perf_counter()
        for i, j in sample:
            operm.match_pair(adj[i], adj[j], absv[i], absv[j], z)
        t_oracle = (time.perf_counter() - t0) / len(sample)
        plan = eperm.match_plan(N)
        print('N=%d M=%d S=%d: %d pairs, cost matrix in %s (%d threads per CTA); host preparation %.3f s; device '
              '%.2f ms (median of %d, min %.2f max %.2f) = %.3g pairs/s; with permutation: %d pairs; oracle %.1f us per '
              'pair (1 process, %d pairs) = %.2f s for all pairs'
              % (N, M, S, n_pairs, plan['path'], plan['threads'], t_prep, dev_ms, len(ms), min(ms), max(ms),
                 n_pairs / (dev_ms * 1e-3), int(d_has.sum().item()), t_oracle * 1e6, len(sample), t_oracle * n_pairs))


if __name__ == '__main__':
    main()
