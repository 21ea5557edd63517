"""GPU time of GDMLPredict.predict against predict_virial, and the B = 1 host-call latency of a periodic model whose cell
changes on every call.

  1. aspirin (N = 21, M = 1000, S = 6) at B = 65 536, CUDA tensors in and out: device time per call (CUDA events),
     the two calls alternated over `--reps` rounds after a warm-up, median reported.
  2. N = 370, M = 500 (S = 6) at B = 256 (the long-descriptor finishing pair), the same way.
  3. B = 1 NumPy in / out (the MD path, CUDA-graph replay) in the aspirin model put in a skewed cell: host time per call
     of predict_virial with a fixed cell, of predict_virial with a new cell on every call, and of set_lattice + predict
     with a new cell on every call (which synchronises the device, and replays the graph).

Prints the results as JSON, with the card's name and power limit; `--out FILE` also writes them to FILE."""

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
    return [float(np.median(t)) for t in times], [float(np.min(t)) for t in times]


def _bulk(name, N, M, S_cfg, sig, B, reps, warmup):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    perms = synth.rotor_swap_group(N, *S_cfg)
    model = synth.random_model(N, M, perms, sig)
    p = sgdml_b200.GDMLPredict(model)
    R = torch.from_numpy(synth.geometries(N, B, 1).reshape(B, -1)).cuda()
    dim_i = 3 * N
    E = torch.empty(B, dtype=torch.float64, device='cuda')
    F = torch.empty((B, dim_i), dtype=torch.float64, device='cuda')
    W = torch.empty((B, 3, 3), dtype=torch.float64, device='cuda')
    E2, F2 = torch.empty_like(E), torch.empty_like(F)
    med, mn = _device_ms([lambda: p.predict(R, out=(E, F)), lambda: p.predict_virial(R, out=(E2, F2, W))], reps, warmup)
    same = bool(torch.equal(E, E2) and torch.equal(F, F2))
    return {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'B': B,
            'predict_ms_median': med[0], 'predict_virial_ms_median': med[1],
            'predict_ms_min': mn[0], 'predict_virial_ms_min': mn[1],
            'overhead_pct_median': 100.0 * (med[1] / med[0] - 1.0), 'E_F_bit_identical': same}


def _latency(calls):
    import sgdml_b200
    import predict_checks as pc  # noqa: F401  (tests/ on the path: skewed_cell)
    from sgdml_b200 import synth

    N, M = 21, 1000
    perms = synth.rotor_swap_group(N, 1, 1)
    lat = pc.skewed_cell(N) * 1.6
    model = synth.random_model(N, M, perms, 20)
    model['lattice'] = lat
    R1 = synth.geometries(N, 1, 1).reshape(1, -1)
    cells = [(1.0 + 1e-4 * (i % 50)) * lat for i in range(calls)]
    inv = [np.linalg.inv(c) for c in cells]
    out = {}
    p = sgdml_b200.GDMLPredict(model)
    for _ in range(20):
        p.predict_virial(R1)
    t0 = time.perf_counter()
    for _ in range(calls):
        p.predict_virial(R1)
    out['predict_virial_fixed_cell_us'] = (time.perf_counter() - t0) / calls * 1e6
    for i in range(20):
        p.predict_virial(R1, lattice=cells[i])
    t0 = time.perf_counter()
    for i in range(calls):
        p.predict_virial(R1, lattice=cells[i])
    out['predict_virial_new_cell_us'] = (time.perf_counter() - t0) / calls * 1e6
    from sgdml_b200 import _lib

    L = _lib.lib()
    n = max(calls // 10, 20)
    for _ in range(20):
        p.predict(R1)
    t0 = time.perf_counter()
    for _ in range(calls):
        p.predict(R1)
    out['predict_fixed_cell_us'] = (time.perf_counter() - t0) / calls * 1e6
    t0 = time.perf_counter()
    for i in range(n):
        c = np.ascontiguousarray(cells[i])
        ci = np.ascontiguousarray(inv[i])
        _lib.check(L.sgdml_b200_model_set_lattice(p._handle, _lib.ptr(c), _lib.ptr(ci)), 'set_lattice')
        p.predict(R1)
    out['set_lattice_plus_predict_new_cell_us'] = (time.perf_counter() - t0) / n * 1e6
    out['calls'] = calls
    out['set_lattice_calls'] = n
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--calls', type=int, default=2000)
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))
    from sgdml_b200 import _lib

    _lib.require_gpu()
    res = {'gpu': _gpu_info()}
    res['aspirin'] = _bulk('aspirin', 21, 1000, (1, 1), 20, 65536, a.reps, a.warmup)
    print(json.dumps(res['aspirin']), flush=True)
    res['n370'] = _bulk('N370', 370, 500, (1, 1), 20, 256, a.reps, a.warmup)
    print(json.dumps(res['n370']), flush=True)
    res['latency_b1'] = _latency(a.calls)
    print(json.dumps(res['latency_b1']), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
