"""Device time of GDMLPredict.predict against predict_hvp, and of the autograd paths of torchtools.GDMLTorchPredict.

For the aspirin shapes (N = 21, M = 1000, S = 6: the fused predictor, D = 210 <= 256) and the ac-ala3-nhme shapes
(N = 42, M = 2000, S = 243: the GEMM-composed predictor, D = 861), synthetic models (synth.random_model):
  1. predict and predict_hvp at B = 1, 64 and 4096, CUDA tensors in and out, alternated over `--reps` rounds after a
     warm-up, CUDA events around each call, median reported;
  2. GDMLTorchPredict forward plus the backward of a force-matching loss ((F - F0)^2).sum() at B = 64 (and 4096 for
     aspirin): one predict and one HVP;
  3. one full 3N-row Hessian of one geometry through the batched-identity form (one engine call of B = 3N).
The flop count of the HVP's four GEMMs, 4 x 2 (2 B S) Mpad DS, comes from the shapes.  Prints JSON with the card's name,
power limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def _gpu_info():
    try:
        return subprocess.check_output(
            ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], text=True
        ).strip()
    except Exception as e:  # noqa: BLE001
        return 'unknown (%s)' % e


def _device_ms(fns, reps, warmup):
    """Median device ms per call of each fn, the fns alternated within every round."""
    import torch

    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[i].append(a.elapsed_time(b))
    return [float(np.median(t)) for t in times]


def _layout(N, M):
    """(D, DP, DS, Mpad) of sgdml_b200_model_create."""
    D = N * (N - 1) // 2
    for DP, BM in ((40, 32), (72, 32), (112, 16), (160, 16), (224, 16), (256, 8)):
        if D <= DP:
            break
    else:
        DP, BM = (D + 7) // 8 * 8, 8
    return D, DP, DP + 4, (M + BM - 1) // BM * BM


def _workload(name, batches, loss_batches, reps, warmup):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth
    from sgdml_b200.torchtools import GDMLTorchPredict

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    S = int(perms.shape[0])
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    D, DP, DS, Mpad = _layout(N, M)
    p = sgdml_b200.GDMLPredict(model)
    res = {'workload': name, 'N': N, 'M': M, 'S': S, 'D': D, 'Mpad': Mpad, 'DS': DS, 'rows': []}
    Rall = torch.from_numpy(synth.geometries(N, max(batches), 1, r0=r0).reshape(-1, 3 * N)).cuda()
    Vall = torch.from_numpy(np.random.default_rng(2).standard_normal(Rall.shape)).cuda()
    for B in batches:
        R, V = Rall[:B].contiguous(), Vall[:B].contiguous()
        E, F, HV = (torch.empty(B, dtype=torch.float64, device='cuda'), torch.empty_like(R), torch.empty_like(R))
        med = _device_ms([lambda: p.predict(R, out=(E, F)), lambda: p.predict_hvp(R, V, out=HV)], reps, warmup)
        gflop = 4 * 2.0 * (2 * B * S) * Mpad * DS / 1e9
        row = {'B': B, 'predict_ms': med[0], 'predict_hvp_ms': med[1], 'hvp_over_predict': med[1] / med[0],
               'hvp_gemm_gflop': gflop, 'hvp_gemm_tflops_over_call': gflop / med[1]}  # GFLOP / ms = TFLOP/s
        print(json.dumps(row), flush=True)
        res['rows'].append(row)
    mod = GDMLTorchPredict(model)
    res['torch_loss'] = []
    for B in loss_batches:
        R = Rall[:B].reshape(B, N, 3).clone().requires_grad_()
        F0 = torch.zeros(B, N, 3, dtype=torch.float64, device='cuda')

        def step():
            _, F = mod(R)
            return torch.autograd.grad(((F - F0) ** 2).sum(), R)

        med = _device_ms([step], reps, warmup)
        row = {'B': B, 'forward_plus_force_loss_backward_ms': med[0]}
        print(json.dumps(row), flush=True)
        res['torch_loss'].append(row)
    Rb = Rall[:1].reshape(1, N, 3).expand(3 * N, N, 3).clone().requires_grad_()
    eye = torch.eye(3 * N, dtype=torch.float64, device='cuda').reshape(3 * N, N, 3)

    def hessian():
        _, Fb = mod(Rb)
        return torch.autograd.grad(Fb, Rb, grad_outputs=-eye)

    res['hessian_batched_identity_ms'] = _device_ms([hessian], reps, warmup)[0]
    res['hessian_rows'] = 3 * N
    print(json.dumps({'hessian_rows': 3 * N, 'ms': res['hessian_batched_identity_ms']}), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    from sgdml_b200 import _lib

    _lib.require_gpu()
    res = {'gpu': _gpu_info()}
    print(json.dumps(res), flush=True)
    res['aspirin'] = _workload('aspirin', (1, 64, 4096), (64, 4096), a.reps, a.warmup)
    res['ac-ala3-nhme'] = _workload('ac-ala3-nhme', (1, 64, 4096), (64,), a.reps, a.warmup)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
