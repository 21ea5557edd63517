"""CPU checks of the numerical claims behind the int8 (FP64-via-INT8) trailing updates
(DESIGN.md section 7, tools/ozaki_study.py): exact integer emulation, no GPU."""

import importlib.util
import os

import numpy as np

from conftest import ROOT

_spec = importlib.util.spec_from_file_location('ozaki_study', os.path.join(ROOT, 'tools', 'ozaki_study.py'))
oz = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(oz)


def test_split_is_error_free_up_to_the_last_slice():
    rng = np.random.default_rng(0)
    A = rng.standard_normal((37, 50)) * np.exp2(rng.integers(-30, 30, size=(37, 1)).astype(np.float64))
    for s in (3, 5, 8):
        e, sl = oz.split_rows(A, s)
        assert np.all(np.abs(sl) <= 64) and np.all(sl == np.rint(sl))  # int8 range, integers
        rec = sum(sl[p] * 2.0 ** (-oz.BITS * (p + 1)) for p in range(s)) * np.exp2(e)[:, None]
        # remainder below half a unit of the last slice, relative to the row's power-of-two scale
        assert np.all(np.abs(rec - A) <= 0.5 * 2.0 ** (-oz.BITS * s) * np.exp2(e)[:, None] * (1 + 1e-12))


def test_gemm_error_falls_by_seven_bits_per_slice():
    rng = np.random.default_rng(1)
    A, B = rng.standard_normal((96, 128)), rng.standard_normal((80, 128))
    ref = A @ B.T
    errs = [np.max(np.abs(oz.ozaki_gemm_nt(A, B, s) - ref)) / np.max(np.abs(ref)) for s in (4, 5, 6, 7, 8)]
    assert errs[3] < 1e-13 and errs[4] < 1e-14  # S = 7, 8
    for lo, hi in zip(errs[1:4], errs[:3]):
        assert lo < hi / 16  # at least 4 of the 7 bits per extra slice show up in the max norm


def test_cholesky_with_seven_slices_matches_fp64_on_an_ill_conditioned_system():
    rng = np.random.default_rng(2)
    n = 600
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    A = (Q * np.logspace(0, -9, n)) @ Q.T  # condition 1e9
    A = 0.5 * (A + A.T)
    y = rng.standard_normal(n)
    L_ref = oz.blocked_cholesky(A, 128, lambda W, V: W @ V.T)
    L7 = oz.blocked_cholesky(A, 128, lambda W, V: oz.ozaki_gemm_nt(W, V, 7))
    import scipy.linalg

    x_ref = scipy.linalg.cho_solve((L_ref, True), y)
    x7 = scipy.linalg.cho_solve((L7, True), y)
    resid = np.linalg.norm(A @ x7 - y) / np.linalg.norm(y)
    resid_ref = np.linalg.norm(A @ x_ref - y) / np.linalg.norm(y)
    assert resid < 50 * max(resid_ref, 1e-12)
