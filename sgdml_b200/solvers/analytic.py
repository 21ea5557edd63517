"""``Analytic`` -- closed-form solver (reference sgdml/solvers/analytic.py:37-159) on the H100.

Assembly writes -K straight into HBM (scale = -1, analytic.py:65), lam is added to the
diagonal, and the FP64 Cholesky factorisation + two triangular solves run on the device
(analytic.py:82-99).  A non-positive-definite matrix surfaces as
``np.linalg.LinAlgError('... not positive definite')`` exactly like SciPy's, so callers'
``except`` clauses keep working; the reference's LU fallback (analytic.py:101-114) is then
run on the host from a freshly assembled matrix.
"""

import logging
import timeit
from functools import partial

import numpy as np

from .. import _lib

DONE = 1
NOT_DONE = 0


class Analytic(object):
    def __init__(self, gdml_train, desc, callback=None):
        self.log = logging.getLogger(__name__)
        self.gdml_train = gdml_train
        self.desc = desc
        self.callback = callback
        self.timings = {}

    def solve(self, task, R_desc, R_d_desc, tril_perms_lin, y):
        """analytic.py:49-151 -> alphas (3NM,)."""
        import torch

        sig = task['sig']
        lam = task['lam']
        use_E_cstr = bool(task.get('use_E_cstr', False))

        n_train = R_d_desc.shape[0]
        if self.callback is not None:
            self.callback = partial(self.callback, disp_str='Assembling kernel matrix')
            self.callback(0, 100)

        # K lives in HBM from assembly to the factorisation; its allocation (a 32 GB cudaMalloc at
        # BASELINE config 2) is kept out of the assembly timing
        n = n_train * 3 * self.desc.n_atoms
        t_alloc = timeit.default_timer()
        if not use_E_cstr:
            ldk = (n + 1) // 2 * 2
            K = self.gdml_train._kernel_matrix_buffer(n, ldk)  # kept across the tasks of a sigma grid
        torch.cuda.synchronize()
        t_alloc = timeit.default_timer() - t_alloc
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        if use_E_cstr:  # M extra rows and columns (train.py:234-300, analytic.py:53-73)
            K = self.gdml_train._assemble_kernel_mat_ecstr_device(R_desc, R_d_desc, tril_perms_lin, sig, scale=-1.0)
            n = n + n_train
        else:
            K, n = self.gdml_train._assemble_kernel_mat_device(
                R_desc, R_d_desc, tril_perms_lin, sig, scale=-1.0, out=K
            )  # analytic.py:65 (flip sign to make convex)
        ev[1].record()

        if self.callback is not None:
            self.callback = partial(self.callback, disp_str='Solving linear system (Cholesky factorization)')
            self.callback(NOT_DONE)

        start = timeit.default_timer()
        y = np.ascontiguousarray(y, dtype=np.float64)
        alphas = np.empty(n)
        try:
            _lib.check(
                _lib.lib().sgdml_b200_solve_analytic(
                    K.data_ptr(), n, K.shape[1], float(lam), _lib.ptr(y), _lib.ptr(alphas), _lib.current_stream()
                ),
                'solve_analytic',
            )
        except np.linalg.LinAlgError:
            # The factorisation overwrote K: assemble it again.  If the trailing updates ran on int8 slices (selected
            # with SGDML_B200_OZAKI_SLICES / sgdml_b200_set_solve_slices), whose 2e-14 error could push a borderline
            # matrix over the edge, first retry with all-FP64 ones; then the reference's fallback, a solver that
            # makes fewer assumptions (host LU, analytic.py:101-114).  A failed FP64 factorisation is deterministic
            # and is not repeated.
            import scipy.linalg

            def reassemble():
                self.gdml_train._K_buf = None
                if use_E_cstr:
                    return self.gdml_train._assemble_kernel_mat_ecstr_device(R_desc, R_d_desc, tril_perms_lin, sig, scale=-1.0)
                return self.gdml_train._assemble_kernel_mat_device(R_desc, R_d_desc, tril_perms_lin, sig, scale=-1.0)[0]

            del K
            K = reassemble()
            L = _lib.lib()
            solved = False
            if L.sgdml_b200_get_solve_slices() > 0:
                L.sgdml_b200_set_solve_slices(0)
                try:
                    _lib.check(
                        L.sgdml_b200_solve_analytic(K.data_ptr(), n, K.shape[1], float(lam), _lib.ptr(y), _lib.ptr(alphas), _lib.current_stream()),
                        'solve_analytic',
                    )
                    solved = True
                    self.log.warning('Cholesky factorisation with int8-sliced trailing updates failed; the FP64 factorisation succeeded.')
                except np.linalg.LinAlgError:
                    del K
                    K = reassemble()
                finally:
                    L.sgdml_b200_set_solve_slices(-1)
            if not solved:
                self.log.warning('Cholesky factorisation failed (matrix not positive definite); falling back to LU.')
                Kh = K[:, :n].cpu().numpy()
                Kh[np.diag_indices_from(Kh)] += lam
                alphas = -scipy.linalg.solve(Kh, y, overwrite_a=True, check_finite=False)
        ev[2].record()
        torch.cuda.synchronize()
        self.timings = {
            'assemble_s': ev[0].elapsed_time(ev[1]) * 1e-3,
            'solve_s': ev[1].elapsed_time(ev[2]) * 1e-3,
            'alloc_s': t_alloc,
        }
        t_free = timeit.default_timer()
        del K  # (the buffer itself stays with the GDMLTrain instance for the next task; release_buffers() frees it)
        torch.cuda.synchronize()
        self.timings['free_s'] = timeit.default_timer() - t_free

        if self.callback is not None:
            dur_s = timeit.default_timer() - start
            self.callback(
                DONE,
                disp_str='Training on {:,} points'.format(n_train),
                sec_disp_str='took {:.1f} s'.format(dur_s) if dur_s >= 0.1 else '',
            )
        return alphas

    @staticmethod
    def est_memory_requirement(n_train, n_atoms):
        """Device bytes: K once (factorised in place; the reference needs ~3x, analytic.py:153-159)
        plus the panel workspace and vectors."""
        n = n_train * 3 * n_atoms
        return n * n * 8 + n * 1024 * 8 + 4 * n * 8
