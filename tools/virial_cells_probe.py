"""Cost of one cell per geometry in GDMLPredict.predict_virial, on a 21-atom, M = 1000, S = 6 periodic model.

  1. B = 65 536 CUDA tensors in and out: time per call between CUDA events (host work inside the call included) with
     one (3, 3) cell against a (B, 3, 3) stack of cells, and against sgdml_b200_predict_virial_cells called directly
     with inverses computed once; the calls alternated over `--reps` rounds after a warm-up, median and min reported,
     with the host time of np.linalg.inv on the B cells.
  2. B = 1, 4 and 16 NumPy in / out (the CUDA-graph path): host time per call with new per-geometry cells on every call,
     against the single-cell call with a new cell on every call.
  3. 1000 frames, each in its own cell: one per-geometry-cell call against 1000 single-cell B = 1 calls (host time).

Prints the results as JSON, with the card's name and power limit; `--out FILE` also writes them to FILE."""

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402

from virial_probe import _device_ms, _gpu_info  # noqa: E402


def _model():
    import predict_checks as pc

    from sgdml_b200 import synth

    N, M = 21, 1000
    perms = synth.rotor_swap_group(N, 1, 1)
    model = synth.random_model(N, M, perms, 20)
    lat = pc.skewed_cell(N) * 1.6
    model['lattice'] = lat
    return N, model, lat


def _cells(lat, n, seed):
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(np.stack([(np.eye(3) + 0.02 * rng.uniform(-1, 1, (3, 3))) @ lat for _ in range(n)]))


def _bulk(p, N, lat, B, reps, warmup):
    import torch

    from sgdml_b200 import synth

    R = torch.from_numpy(synth.geometries(N, B, 1).reshape(B, -1)).cuda()
    cells = _cells(lat, B, 2)
    eq = np.ascontiguousarray(np.repeat(lat[None], B, axis=0))
    outs = [(torch.empty(B, dtype=torch.float64, device='cuda'), torch.empty((B, 3 * N), dtype=torch.float64, device='cuda'),
             torch.empty((B, 3, 3), dtype=torch.float64, device='cuda')) for _ in range(3)]
    # the C call with the inverses computed once: what the engine itself adds per geometry, without the
    # np.linalg.inv of B cells that predict_virial does on every call
    from sgdml_b200 import _lib

    L = _lib.lib()
    inv = np.ascontiguousarray(np.linalg.inv(cells))

    def c_call():
        _lib.check(L.sgdml_b200_predict_virial_cells(p._handle, R.data_ptr(), B, _lib.ptr(cells), _lib.ptr(inv),
                                                     outs[1][0].data_ptr(), outs[1][1].data_ptr(),
                                                     outs[1][2].data_ptr(), _lib.current_stream()), 'cells')

    med, mn = _device_ms([lambda: p.predict_virial(R, lattice=lat, out=outs[0]),
                          lambda: p.predict_virial(R, lattice=cells, out=outs[1]), c_call], reps, warmup)
    t0 = time.perf_counter()
    for _ in range(5):
        np.linalg.inv(cells)
    inv_ms = (time.perf_counter() - t0) / 5 * 1e3
    p.predict_virial(R, lattice=eq, out=outs[2])
    torch.cuda.synchronize()
    same = all(bool(torch.equal(a, b)) for a, b in zip(outs[0], outs[2]))
    return {'B': B, 'one_cell_ms_median': med[0], 'cell_per_geometry_ms_median': med[1],
            'cell_per_geometry_c_abi_precomputed_inverses_ms_median': med[2], 'one_cell_ms_min': mn[0],
            'cell_per_geometry_ms_min': mn[1], 'cell_per_geometry_c_abi_ms_min': mn[2],
            'host_inv_of_B_cells_ms': inv_ms, 'diff_pct_median': 100.0 * (med[1] / med[0] - 1.0),
            'c_abi_diff_pct_median': 100.0 * (med[2] / med[0] - 1.0), 'equal_cells_bit_identical': same}


def _latency(p, N, lat, calls):
    from sgdml_b200 import synth

    out = {}
    for B in (1, 4, 16):
        R = synth.geometries(N, B, 3).reshape(B, -1)
        stacks = [_cells(lat, B, 10 + i) for i in range(50)]
        singles = [s[0] for s in stacks]
        for i in range(20):
            p.predict_virial(R, lattice=stacks[i % 50])
            p.predict_virial(R, lattice=singles[i % 50])
        t0 = time.perf_counter()
        for i in range(calls):
            p.predict_virial(R, lattice=stacks[i % 50])
        out['B%d_cell_per_geometry_us' % B] = (time.perf_counter() - t0) / calls * 1e6
        t0 = time.perf_counter()
        for i in range(calls):
            p.predict_virial(R, lattice=singles[i % 50])
        out['B%d_one_new_cell_us' % B] = (time.perf_counter() - t0) / calls * 1e6
    out['calls'] = calls
    return out


def _frames(p, N, lat, n=1000, reps=5):
    from sgdml_b200 import synth

    R = synth.geometries(N, n, 4).reshape(n, -1)
    cells = _cells(lat, n, 5)
    p.predict_virial(R, lattice=cells)
    for i in range(20):
        p.predict_virial(R[i : i + 1], lattice=cells[i])
    one, many = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        _, _, W1 = p.predict_virial(R, lattice=cells)
        one.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        Ws = [p.predict_virial(R[i : i + 1], lattice=cells[i])[2] for i in range(n)]
        many.append(time.perf_counter() - t0)
    err = float(np.max(np.abs(np.concatenate(Ws) - W1)) / np.max(np.abs(W1)))
    return {'frames': n, 'one_call_ms_median': 1e3 * float(np.median(one)),
            'single_cell_calls_ms_median': 1e3 * float(np.median(many)), 'max_rel_W_difference': err}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--calls', type=int, default=2000)
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    N, model, lat = _model()
    p = sgdml_b200.GDMLPredict(model)
    res = {'gpu': _gpu_info()}
    res['bulk'] = _bulk(p, N, lat, 65536, a.reps, a.warmup)
    print(json.dumps(res['bulk']), flush=True)
    res['latency'] = _latency(p, N, lat, a.calls)
    print(json.dumps(res['latency']), flush=True)
    res['frames'] = _frames(p, N, lat)
    print(json.dumps(res['frames']), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
