"""Per-call timing of GDMLPredict.predict (device-resident inputs): GPU time (events) and host time.

    python tools/predict_probe.py [WORKLOADS] [B]

WORKLOADS is a comma-separated list of synth.CONFIGS names or atom counts; an atom count N times a synthetic
molecule with M = 1000 training points and S = 6 permutations (D = N (N - 1) / 2 picks the predictor's tile class:
9, 12, 15, 18, 21, 23 cover all six)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import sgdml_b200
from sgdml_b200 import synth, _lib
wls = (sys.argv[1] if len(sys.argv) > 1 else 'ethanol').split(',')
B = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
for wl in wls:
    if wl.isdigit():
        cfg = dict(n_atoms=int(wl), n_train=1000, n_rotors=1, n_swaps=1, sig=20)
        wl = 'N%s (D %d)' % (wl, int(wl) * (int(wl) - 1) // 2)
    else:
        cfg = synth.CONFIGS[wl]
    perms = synth.rotor_swap_group(cfg['n_atoms'], cfg['n_rotors'], cfg['n_swaps'])
    model = synth.random_model(cfg['n_atoms'], cfg['n_train'], perms, cfg['sig'])
    p = sgdml_b200.GDMLPredict(model)
    R = torch.from_numpy(synth.geometries(cfg['n_atoms'], B, 1).reshape(B, -1)).cuda()
    for _ in range(3): p.predict(R)
    torch.cuda.synchronize()
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(11)]
    host = []
    evs[0].record()
    for i in range(10):
        t0 = time.perf_counter(); p.predict(R); host.append((time.perf_counter() - t0) * 1e3); evs[i + 1].record()
    torch.cuda.synchronize()
    gpu = [evs[i].elapsed_time(evs[i + 1]) for i in range(10)]
    print(wl, 'B', B, 'M', cfg['n_train'], 'S', len(perms), 'gpu ms per call: median %.3f' % float(np.median(gpu)),
          ['%.2f' % g for g in gpu])
    print('host ms per call', ['%.2f' % h for h in host])
    out = (torch.empty(B, dtype=torch.float64, device='cuda'), torch.empty((B, R.shape[1]), dtype=torch.float64, device='cuda'))
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for i in range(10): p.predict(R, out=out)
    torch.cuda.synchronize(); print('with out=: ms per call %.3f' % ((time.perf_counter() - t0) * 100), flush=True)
    del p
