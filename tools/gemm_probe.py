"""Raw throughput of the DMMA GEMM kernel (C = A B^T) for a few shapes, operands fed by cp.async (variant 0) and by
TMA (variant 3, the default)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sgdml_b200 import _lib
L = _lib.lib()
for (m, n, k) in [(16384, 16384, 128), (16384, 16384, 512), (16384, 16384, 1024), (8192, 8192, 4096)]:
    A = torch.randn(m, k, dtype=torch.float64, device='cuda'); B = torch.randn(n, k, dtype=torch.float64, device='cuda')
    C = torch.zeros(m, n, dtype=torch.float64, device='cuda')
    for v in (0, 3):
        L.sgdml_b200_set_gemm_variant(v)
        for _ in range(2):
            L.sgdml_b200_dgemm_nt(m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), k, 1.0, C.data_ptr(), n, None)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 5
        e0.record()
        for _ in range(reps):
            L.sgdml_b200_dgemm_nt(m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), k, 1.0, C.data_ptr(), n, None)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        print('gemm m=%d n=%d k=%d variant=%d: %.3f ms  %.2f TFLOP/s' % (m, n, k, v, ms, 2.0 * m * n * k / ms * 1e-9), flush=True)
    if k == 512:
        ref = (A[:64] @ B.T)
        C.zero_(); L.sgdml_b200_set_gemm_variant(3)
        L.sgdml_b200_dgemm_nt(m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), k, 0.0, C.data_ptr(), n, None); torch.cuda.synchronize()
        print('check max abs err vs torch:', float((C[:64] - ref).abs().max()))
L.sgdml_b200_set_gemm_variant(3)
