"""Throughput of the wgmma int8-slice GEMM (csrc/ozaki.cu) next to the DMMA GEMM, same shapes.
FP64-equivalent TFLOP/s = 2 m n k / time; the int8 path's time includes slicing both operands."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from sgdml_b200 import _lib

L = _lib.lib()
S = int(os.environ.get('OZ_S', '7'))
for (m, n, k) in [(16384, 16384, 1024), (32768, 32768, 1024), (16384, 16384, 512)]:
    A = torch.randn(m, k, dtype=torch.float64, device='cuda')
    B = torch.randn(n, k, dtype=torch.float64, device='cuda')
    C = torch.zeros(m, n, dtype=torch.float64, device='cuda')
    L.sgdml_b200_dgemm_nt(m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), k, 0.0, C.data_ptr(), n, None)
    torch.cuda.synchronize()
    ref = C[:256, :256].clone()
    C.zero_()
    for tri in (0, 1):
        for rep in range(3):
            L.sgdml_b200_profile_reset()
            L.sgdml_b200_profile_enable(1)
            rc = L.sgdml_b200_ozaki_gemm_nt(m, n, k, 1.0, A.data_ptr(), k, (A if tri else B).data_ptr(), k, C.data_ptr(), n, S, tri, None)
            torch.cuda.synchronize()
            L.sgdml_b200_profile_enable(0)
            assert rc == 0, _lib.last_error()
            ms, sc, ln = ctypes.c_double(), ctypes.c_int64(), ctypes.c_int64()
            L.sgdml_b200_profile_get(3, ctypes.byref(ms), ctypes.byref(sc), ctypes.byref(ln))
            fl = 2.0 * m * n * k * (0.5 if tri else 1.0)
            print('ozaki S=%d m=%d n=%d k=%d tri=%d: gemm-family device time %.3f ms -> %.1f TFLOP/s FP64-equivalent' % (S, m, n, k, tri, ms.value, fl / ms.value * 1e-9), flush=True)
        if not tri:
            err = float((C[:256, :256] / 3.0 - ref).abs().max() / ref.abs().max())
            print('  rel err vs DMMA GEMM (3 accumulated calls / 3): %.2e' % err, flush=True)
        C.zero_()
