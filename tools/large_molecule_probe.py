"""Large-molecule probe at the double-walled nanotube shape of MD22 (synthetic, N = 370, one rotor: S = 3, M = 500).

    python tools/large_molecule_probe.py [--n-atoms 370] [--n-train 500] [--no-train] [--out DIR]

Reports, with the card name and power limit read in the same run:
  * device ms per GDMLPredict.predict call (device tensors) at B = 1 and B = 256, split into the main part (query rows,
    GEMMs, transform) and the finishing step (k_fdesc_gather + k_fdesc_project, profile family 'predict_finish');
  * the finishing step's achieved bandwidth over the bytes it has to move, against the 3.35 TB/s of the H100 SXM;
  * one full K.v (kmatvec_train over all M training points, the operator of every CG iteration);
  * one iterative training run (GDMLTrain.train with the device-memory budget): wall time, CG iterations, whether it
    converged (iterations below maxiter) and the assembly slab workspace of k_assemble_large.
Per-family times come from the engine's profiler (CUDA events around each family's launches; a separate pass from
the end-to-end timing, which runs with the profiler off)."""

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import sgdml_b200  # noqa: E402
from sgdml_b200 import _lib, synth  # noqa: E402

HBM_TBPS = 3.35  # H100 SXM data sheet
ASM_SLAB_BYTES_MAX = 2 << 30  # csrc/assemble.cu


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return 'unknown (%s)' % e


def finish_bytes(N, S, B):
    """Bytes the finishing step has to move for B queries: G read once (S rows of DP), F_desc written and read,
    the query Jacobians gq read (3 D), F written (3 N), the permutation table read once."""
    D = N * (N - 1) // 2
    DP = (D + 7) // 8 * 8
    return B * (S * DP * 8 + 2 * D * 8 + 3 * D * 8 + 3 * N * 8) + S * D * 4


def slab_bytes(N, S, n_sm):
    N3, NN = 3 * N, N * N
    slab = 2 * (NN * 3 + NN) + S * (2 * N3 + 3 * N3 + 2) + NN
    slab = (slab + 1) // 2 * 2 * 8
    n_cta = max(1, min(2 * n_sm, ASM_SLAB_BYTES_MAX // slab))
    return n_cta, slab, n_cta * slab


def time_calls(fn, reps):
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]))


def profiled(fn, reps):
    L = _lib.lib()
    fn()
    torch.cuda.synchronize()
    L.sgdml_b200_profile_reset()
    L.sgdml_b200_profile_enable(1)
    try:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    finally:
        L.sgdml_b200_profile_enable(0)
    return {k: v[0] / reps for k, v in _lib.profile_snapshot().items() if v[0] > 0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n-atoms', type=int, default=370)
    ap.add_argument('--n-train', type=int, default=500)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--no-train', action='store_true')
    ap.add_argument('--out', default=None, help='also write the result as JSON here')
    args = ap.parse_args()
    _lib.require_gpu()
    N, M = args.n_atoms, args.n_train
    perms = synth.rotor_swap_group(N, 1, 0)
    S = len(perms)
    res = {'card': card(), 'n_atoms': N, 'n_train': M, 'n_perms': S, 'D': N * (N - 1) // 2}
    print(res, flush=True)

    model = synth.random_model(N, M, perms, 50)
    p = sgdml_b200.GDMLPredict(model)
    for B in (1, 256):
        R = torch.from_numpy(synth.geometries(N, B, 1).reshape(B, -1)).cuda()
        ms = time_calls(lambda: p.predict(R), args.reps)
        fam = profiled(lambda: p.predict(R), args.reps)
        fin = fam.get('predict_finish', float('nan'))
        gbs = finish_bytes(N, S, B) / (fin * 1e-3) / 1e9
        res['predict_B%d' % B] = {
            'ms_per_call': ms,
            'profiled_ms': fam,
            'finish_ms': fin,
            'main_ms': sum(v for k, v in fam.items() if k != 'predict_finish'),
            'finish_GBps': gbs,
            'finish_share_of_hbm': gbs / (HBM_TBPS * 1e3),
        }
        print('predict B=%d: %.3f ms/call; profiled %s; finishing %.1f GB/s (%.0f %% of %.2f TB/s)'
              % (B, ms, {k: round(v, 3) for k, v in fam.items()}, gbs, 100 * gbs / (HBM_TBPS * 1e3), HBM_TBPS), flush=True)

    # one full K.v: alphas = v, raw force and energy sums on all training points
    x, g = sgdml_b200.desc.Desc(N).from_R(synth.geometries(N, M, 0).reshape(M, -1))
    p.set_R_desc(x)
    p.set_R_d_desc(g)
    p.set_alphas(np.random.default_rng(1).standard_normal(M * 3 * N))
    F = torch.empty((M, 3 * N), dtype=torch.float64, device='cuda')
    res['kv_ms'] = time_calls(lambda: p.kmatvec_train(0, M, out=F), max(3, args.reps // 4))
    print('K.v over M = %d: %.2f ms' % (M, res['kv_ms']), flush=True)
    del p, x, g, F

    if not args.no_train:
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        n_cta, slab, tot = slab_bytes(N, S, n_sm)
        res['asm_slabs'] = {'ctas': n_cta, 'bytes_per_cta': slab, 'bytes': tot}
        task = synth.make_task(N, M, perms, 50)
        np.random.seed(0)
        t = sgdml_b200.GDMLTrain()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m = t.train(task)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        iters = int(m.get('solver_iters', 0))
        maxiter = 3 * N * M * 10
        res['train'] = {
            'solver': m['solver_name'],
            'wall_s': wall,
            'iters': iters,
            'converged': m['solver_name'] == 'analytic' or iters < maxiter,
            'inducing_pts': len(m.get('inducing_pts_idxs', [])) // (3 * N),
            'timings': {k: float(v) for k, v in getattr(t, 'timings', {}).items() if isinstance(v, (int, float))},
        }
        print('train: %s' % res['train'], 'slabs: %d CTAs x %.1f MB = %.2f GB' % (n_cta, slab / 1e6, tot / 1e9), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'large_molecule_probe.json'), 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
