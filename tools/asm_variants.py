"""Assembly kernel variants at BASELINE config 2 (full symmetric matrix) and for a column subset with many
permutations (the Nystroem set-up of config 3), device time per launch."""
import ctypes, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import sgdml_b200
from sgdml_b200 import synth, _lib
from sgdml_b200.desc import Desc, tril_perms_lin
L = _lib.lib()
t = sgdml_b200.GDMLTrain()
def run(name, N, M, perms, sig, cols, variants=(2, 4, 5, 1, 2, 4, 5, 1)):
    R = synth.geometries(N, M, 0).reshape(M, -1)
    x, g = Desc(N).from_R(R)
    lin = tril_perms_lin(perms)
    ref = None
    for v in variants:
        L.sgdml_b200_set_assemble_variant(0)
        L.sgdml_b200_set_assemble_variant(v)
        K, nc = t._assemble_kernel_mat_device(x, g, lin, sig, col_idxs=cols)  # warm-up + allocation
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        t._assemble_kernel_mat_device(x, g, lin, sig, col_idxs=cols, out=K)
        e1.record(); torch.cuda.synchronize()
        if ref is None: ref = K[:256, :nc].clone()
        dev = float((K[:256, :nc] - ref).abs().max() / ref.abs().max())
        print('%s kernel %d: %.2f ms (%.1f GB written, %.0f GB/s), rel dev vs the first: %.1e' % (
            name, v, e0.elapsed_time(e1), K.shape[0] * nc * 8 / 1e9, K.shape[0] * nc * 8 / 1e6 / e0.elapsed_time(e1), dev), flush=True)
        del K
    L.sgdml_b200_set_assemble_variant(0)
perms = synth.rotor_swap_group(21, 1, 1)
run('aspirin M=1000 S=6 full', 21, 1000, perms, 20, None)
perms = synth.rotor_swap_group(42, 5, 0)
n = 3 * 42 * 300
cols = np.sort(np.random.default_rng(0).choice(n, 3000, replace=False))
run('ac-ala3 M=300 S=243 3000 cols', 42, 300, perms, 50, cols)
perms, r0 = synth.config_perms_and_r0('c60')
n = 3 * 60 * 150
cols = np.sort(np.random.default_rng(0).choice(n, 1500, replace=False))
run('c60 M=150 S=120 1500 cols (variant 1 = large-molecule kernel)', 60, 150, perms, 50, cols, variants=(1, 5, 1, 5))
