"""Times sgdml_b200_potrf alone on a random SPD matrix (device resident)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sgdml_b200 import _lib
L = _lib.lib()
n = int(sys.argv[1]) if len(sys.argv) > 1 else 32768
A0 = torch.randn(n, n, dtype=torch.float64, device='cuda'); A0 = A0 @ A0.T; A0 += n * torch.eye(n, dtype=torch.float64, device='cuda')
for rep in range(3):
    A = A0.clone(); torch.cuda.synchronize()
    t0 = time.perf_counter(); rc = L.sgdml_b200_potrf(A.data_ptr(), n, n, None); torch.cuda.synchronize(); dt = time.perf_counter() - t0
    print('potrf n=%d rc=%d  %.4f s  %.2f TFLOP/s' % (n, rc, dt, n ** 3 / 3 / dt * 1e-12), flush=True)
