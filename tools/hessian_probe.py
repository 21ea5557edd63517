"""Device time of GDMLPredict.predict_hessian against the batched-identity HVP form, of the batched Jacobi eigensolver
against torch.linalg.eigh, and of GDMLVibrations.analyse against the finite-difference route.

Synthetic models (synth.random_model) at the ethanol (N = 9), aspirin (N = 21) and ac-ala3-nhme (N = 42) shapes of
synth.CONFIGS, CUDA tensors in and out, CUDA events, the variants alternated within every round, medians reported:
  1. predict_hessian(R) against predict_hvp(R repeated 3N times, the unit vectors), B = 1, 64 and 1024 geometries (fewer
     where the identity form's 3N B rows would not fit); both results must be bit-identical;
  2. sgdml_b200_symeig_batched against torch.linalg.eigh on the same mass-weighted, projected Hessians (n = 27, 63, 126);
  3. analyse() per geometry against 6N central-difference predict calls of one geometry each (ASE's Vibrations).
Prints JSON with the card's name and power limit read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def _gpu_info():
    return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                    '--format=csv,noheader'], text=True).strip()


def _device_ms(fns, reps, warmup):
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


def _workload(name, batches, reps, warmup):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth, vib

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    S = int(perms.shape[0])
    gp = sgdml_b200.GDMLPredict(synth.random_model(N, M, perms, cfg['sig'], r0=r0))
    n = 3 * N
    res = {'workload': name, 'N': N, 'M': M, 'S': S, 'hessian': [], 'symeig': [], 'analyse': None}
    Rall = torch.from_numpy(synth.geometries(N, max(batches), 1, r0=r0).reshape(-1, n)).cuda()
    eye = torch.eye(n, dtype=torch.float64, device='cuda')
    for B in batches:
        R = Rall[:B].contiguous()
        Rrep = R.repeat_interleave(n, 0).contiguous()
        E = eye.repeat(B, 1).contiguous()
        H = gp.predict_hessian(R)
        HV = gp.predict_hvp(Rrep, E)  # row b n + i: column i of -H[b]
        same = bool(torch.equal(H, -HV.reshape(B, n, n).transpose(1, 2)))
        t_h, t_i = _device_ms([lambda: gp.predict_hessian(R), lambda: gp.predict_hvp(Rrep, E)], reps, warmup)
        res['hessian'].append({'B': B, 'hessian_ms': t_h, 'identity_hvp_ms': t_i, 'speedup': t_i / t_h,
                               'bit_identical': same})
        print(json.dumps(res['hessian'][-1]), flush=True)
        del Rrep, E, HV
        torch.cuda.empty_cache()
    masses = np.full(N, 12.0)
    v = sgdml_b200.GDMLVibrations(gp, masses, E_to_eV=1.0, F_to_eV_Ang=1.0)
    from sgdml_b200 import _lib

    X = Rall[:64].reshape(-1, N, 3).contiguous()
    H = gp.predict_hessian(X.reshape(-1, n))
    Hp64 = torch.empty_like(H)
    k = torch.empty(len(X), dtype=torch.int64, device='cuda')
    _lib.check(_lib.lib().sgdml_b200_vib_project(_lib.ptr(H), _lib.ptr(X), _lib.ptr(v._ism), len(X), N, 0,
                                                 _lib.ptr(Hp64), _lib.ptr(k), _lib.current_stream()), 'vib_project')
    for B in (64, 1000):  # the 64 projected Hessians, tiled
        Hp = Hp64.repeat((B + len(X) - 1) // len(X), 1, 1)[:B].contiguous()
        t_j, t_t = _device_ms([lambda: vib.symeig(Hp), lambda: torch.linalg.eigh(Hp)], max(3, reps // 4), 1)
        wj, wt = vib.symeig(Hp)[0], torch.linalg.eigh(Hp)[0]
        dev = float((wj - wt).abs().max() / wt.abs().max())
        res['symeig'].append({'n': n, 'B': B, 'jacobi_ms': t_j, 'torch_eigh_ms': t_t, 'speedup': t_t / t_j,
                              'max_rel_eig_diff': dev})
        print(json.dumps(res['symeig'][-1]), flush=True)
    X1 = Rall[:1].reshape(1, N, 3)
    Xb = Rall[:64].reshape(-1, N, 3)

    def fd():
        x = X1.reshape(1, n)
        for i in range(n):
            for s in (1e-4, -1e-4):
                xp = x.clone()
                xp[0, i] += s
                gp.predict(xp)

    t_a1, t_a64, t_fd = _device_ms([lambda: v.analyse(X1), lambda: v.analyse(Xb), fd], max(3, reps // 4), 1)
    res['analyse'] = {'analyse_1_ms': t_a1, 'analyse_64_ms_per_geometry': t_a64 / len(Xb),
                      'fd_6N_predict_ms_per_geometry': t_fd}
    print(json.dumps(res['analyse']), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    ap.add_argument('--workloads', default='ethanol,aspirin,ac-ala3-nhme')
    a = ap.parse_args()
    info = _gpu_info()
    print(info, flush=True)
    # the identity form holds 3N B geometries: B = 1024 at N = 42 is 129k HVP rows of 243 permutations, beyond memory
    batches = {'ethanol': (1, 64, 1024), 'aspirin': (1, 64, 1024), 'ac-ala3-nhme': (1, 8)}
    out = {'gpu': info, 'results': [_workload(w, batches[w], a.reps, a.warmup) for w in a.workloads.split(',')]}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s)


if __name__ == '__main__':
    main()
