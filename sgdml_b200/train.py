"""``GDMLTrain`` -- the reference's training API (sgdml/train.py:305-1258) on the H100 engine.

Hot path only: ``train(task)``, ``create_model``, ``_recov_int_const`` and
``_assemble_kernel_mat`` keep the reference's names, arguments and model/.npz layout
(train.py:793-830).  Task creation / sampling / permutation discovery stay the reference's
own host code (SURVEY.md section 2 rows 12-13, out of scope): a task dict produced by
``sgdml.train.GDMLTrain.create_task`` is a valid input here.

K is assembled directly in HBM, negated and regularised in place and factorised there; the
reference's torch engine copies every block-column to the host (torchtools.py:233) and
always factorises on the CPU (analytic.py:94).
"""

import logging
import timeit

import numpy as np

from . import _lib
from .desc import Desc, tril_perms_lin as _tril_perms_lin
from .predict import GDMLPredict
from .solvers.analytic import Analytic
from .solvers.iterative import Iterative

__version__ = '0.1.0'


def _torch():
    import torch

    return torch


def labels(task, use_E_cstr):
    """The normalised label vector train() solves for (train.py:939-947): y = F_train.ravel() / std, with energy
    constraints [F_train.ravel(); -E_train + mean(E_train)] / std.  Returns (y, std, mean(E_train) or None)."""
    y = np.asarray(task['F_train'], dtype=np.float64).ravel().copy()
    E_train_mean = None
    if use_E_cstr:
        E_train = np.asarray(task['E_train'], dtype=np.float64).ravel().copy()
        E_train_mean = np.mean(E_train)
        y = np.hstack((y, -E_train + E_train_mean))
    y_std = np.std(y)
    y /= y_std
    return y, y_std, E_train_mean


class GDMLTrain(object):
    def __init__(self, max_memory=None, max_processes=None, use_torch=False):
        """train.py:306-361.  `max_memory` [GB] caps the device memory the analytic solver
        may use (default: what is free on the current GPU); `max_processes` / `use_torch`
        are accepted for signature compatibility."""
        self.log = logging.getLogger(__name__)
        _lib.require_gpu()
        self._max_memory = max_memory
        self._max_processes = max_processes
        self._use_torch = use_torch
        # Set to True when EVERY rank of an initialised torch.distributed job calls train() with the same task: the
        # ranks then agree on the solver and its memory budget (one all-reduce) and the iterative solver shards its
        # work over them (row-sharded Nystroem factor and K.v, SURVEY.md section 8e).  False (default): this process
        # trains alone and issues no collective, whatever torch.distributed's state (e.g. rank 0 of a benchmark
        # trains while the other ranks wait for the coefficients).
        self.distributed = False
        # Residency across the tasks of a sigma grid (`sgdml all` retrains the same points for several length scales
        # with ONE GDMLTrain instance, cli.py:802-806, 923-932, 981-1083): descriptors and Jacobians are
        # sigma-independent and stay on the device, the kernel-matrix buffer (31.8 GB at BASELINE config 2) and the
        # factorisation workspaces are allocated once.  release_buffers() drops them.
        self._desc_cache = {}
        self._K_buf = None
        self.cache_stats = {'desc_hits': 0, 'desc_misses': 0, 'K_reused': 0, 'K_allocated': 0}

    def release_buffers(self):
        """Frees the device buffers kept between train() calls (descriptor cache, K, factorisation workspaces)."""
        self._desc_cache.clear()
        self._K_buf = None
        _lib.lib().sgdml_b200_release_workspaces()
        _torch().cuda.empty_cache()

    def _descriptors(self, desc, R, lat_and_inv):
        """R_desc, R_d_desc of the training geometries as host arrays AND device tensors, cached by content."""
        import hashlib

        torch = _torch()
        h = hashlib.blake2b(R.tobytes(), digest_size=16)
        if lat_and_inv is not None:
            h.update(np.ascontiguousarray(lat_and_inv[0]).tobytes())
        key = (R.shape, h.hexdigest())
        hit = self._desc_cache.get(key)
        if hit is not None:
            self.cache_stats['desc_hits'] += 1
            return hit
        self.cache_stats['desc_misses'] += 1
        R_desc, R_d_desc = desc.from_R(R, lat_and_inv=lat_and_inv)  # train.py:926-935
        if R.shape[0] == 1:
            R_desc, R_d_desc = R_desc[None], R_d_desc[None]
        entry = (R_desc, R_d_desc, torch.from_numpy(R_desc).cuda(), torch.from_numpy(R_d_desc).cuda())
        if len(self._desc_cache) >= 4:  # a handful of training sets at most
            self._desc_cache.pop(next(iter(self._desc_cache)))
        self._desc_cache[key] = entry
        return entry

    def _kernel_matrix_buffer(self, n_rows, ldk):
        """A (n_rows, ldk) float64 CUDA tensor, reused between train() calls of the same size."""
        torch = _torch()
        if self._K_buf is not None and tuple(self._K_buf.shape) == (n_rows, ldk):
            self.cache_stats['K_reused'] += 1
            return self._K_buf
        self._K_buf = None  # free the old one first
        self._K_buf = torch.empty((n_rows, ldk), dtype=torch.float64, device='cuda')
        self.cache_stats['K_allocated'] += 1
        return self._K_buf

    # ------------------------------------------------------------------ model assembly
    def create_model(self, task, solver, R_desc, R_d_desc, tril_perms_lin, std, alphas_F, alphas_E=None):
        """train.py:727-832: same keys, shapes and dtypes as the reference model dict."""
        n_train, dim_d = R_d_desc.shape[:2]
        n_atoms = int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        desc = Desc(n_atoms, max_processes=self._max_processes)
        dim_i = desc.dim_i
        R_d_desc_alpha = desc.d_desc_dot_vec(R_d_desc, alphas_F.reshape(-1, dim_i))  # train.py:791

        model = {
            'type': 'm',
            'code_version': __version__,
            'dataset_name': task['dataset_name'],
            'dataset_theory': task['dataset_theory'],
            'solver_name': solver,
            'z': task['z'],
            'idxs_train': task['idxs_train'],
            'md5_train': task['md5_train'],
            'idxs_valid': task['idxs_valid'],
            'md5_valid': task['md5_valid'],
            'n_test': 0,
            'md5_test': None,
            'f_err': {'mae': np.nan, 'rmse': np.nan},
            'R_desc': R_desc.T,  # train.py:807 (transposed)
            'R_d_desc_alpha': R_d_desc_alpha,
            'c': 0.0,
            'std': std,
            'sig': task['sig'],
            'lam': task['lam'],
            'alphas_F': alphas_F,
            'perms': task['perms'],
            'tril_perms_lin': tril_perms_lin,
            'use_E': task['use_E'],
        }
        if task['use_E']:
            model['e_err'] = {'mae': np.nan, 'rmse': np.nan}
            if task['use_E_cstr']:
                model['alphas_E'] = alphas_E
        if 'lattice' in task:
            model['lattice'] = task['lattice']
        if 'r_unit' in task and 'e_unit' in task:
            model['r_unit'] = task['r_unit']
            model['e_unit'] = task['e_unit']
        return model

    # ------------------------------------------------------------------ training
    def train(self, task, save_progr_callback=None, callback=None):
        """train.py:836-1088.  Returns the model dict."""
        t_all = timeit.default_timer()
        task = dict(task)
        use_E_cstr = bool(task.get('use_E', False)) and bool(task.get('use_E_cstr', False))
        task['use_E_cstr'] = use_E_cstr

        n_train, n_atoms = task['R_train'].shape[:2]
        desc = Desc(n_atoms, max_processes=self._max_processes)

        tril_perms_lin = _tril_perms_lin(task['perms'])  # train.py:897-904

        lat_and_inv = None
        if 'lattice' in task:  # train.py:906-911
            lat = np.ascontiguousarray(task['lattice'], dtype=np.float64)
            lat_and_inv = (lat, np.ascontiguousarray(np.linalg.inv(lat)))
        R = np.ascontiguousarray(task['R_train'], dtype=np.float64).reshape(n_train, -1)
        R_desc, R_d_desc, R_desc_dev, R_d_desc_dev = self._descriptors(desc, R, lat_and_inv)
        self._dev_views = {id(R_desc): R_desc_dev, id(R_d_desc): R_d_desc_dev}  # device twins of the host arrays

        y, y_std, E_train_mean = labels(task, use_E_cstr)

        t_desc = timeit.default_timer() - t_all
        # solver choice by memory, like train.py:949-975 -- but against DEVICE memory
        est_bytes_analytic = Analytic.est_memory_requirement(n_train, n_atoms)
        free_bytes, _total = _torch().cuda.mem_get_info()
        max_bytes = free_bytes if self._max_memory is None else min(free_bytes, self._max_memory * 1024**3)
        # several ranks must take the SAME decision (the iterative path issues collectives the analytic one
        # never joins) and derive the same number of inducing points: agree on the smallest budget
        if self.distributed:
            from . import dist as sdist

            max_bytes = sdist.all_reduce_min_scalar(max_bytes)
        # with energy constraints the iterative solver works on the (3NM + M)-square system [forces; energies], as the
        # reference's does (iterative.py:183-204, 372-379, 685-698)
        use_analytic_solver = est_bytes_analytic < max_bytes

        solver_keys = {}
        if use_analytic_solver:
            analytic = Analytic(self, desc, callback=callback)
            alphas = analytic.solve(task, R_desc, R_d_desc, tril_perms_lin, y)
            self.timings = dict(analytic.timings)
        else:
            # the Nystroem factor (n x m, the dominant term of iterative.py:845-866) is row-sharded over the ranks of a
            # distributed run, so the budget that sizes the inducing set is the ranks' memory together
            iter_bytes = max_bytes
            if self.distributed:
                import torch.distributed as tdist

                if tdist.is_available() and tdist.is_initialized():
                    iter_bytes = max_bytes * tdist.get_world_size()
            iterative = Iterative(
                self, desc, iter_bytes / 1024**3, self._max_processes, self._use_torch, callback=callback
            )
            (
                alphas,
                solver_keys['solver_tol'],
                solver_keys['solver_iters'],
                solver_keys['solver_resid'],
                train_rmse,
                solver_keys['inducing_pts_idxs'],
                is_conv,
            ) = iterative.solve(task, R_desc, R_d_desc, tril_perms_lin, y, y_std, save_progr_callback=save_progr_callback)
            solver_keys['norm_y_train'] = np.linalg.norm(y)  # train.py:1030
            self.timings = dict(iterative.timings)
            if not is_conv:
                self.log.warning('Iterative solver did not converge! (train.py:1032-1052)')

        t0 = timeit.default_timer()
        alphas_F, alphas_E = alphas, None
        if use_E_cstr:  # train.py:1052-1056
            alphas_E = alphas[-n_train:]
            alphas_F = alphas[:-n_train]
        model = self.create_model(
            task, 'analytic' if use_analytic_solver else 'cg', R_desc, R_d_desc, tril_perms_lin, y_std, alphas_F,
            alphas_E=alphas_E,
        )
        model.update(solver_keys)
        t1 = timeit.default_timer()
        if model['use_E']:  # train.py:1071-1086: with energy constraints c is the mean of the training energies
            model['c'] = (
                self._recov_int_const(model, task, R_desc=R_desc, R_d_desc=R_d_desc) if E_train_mean is None else E_train_mean
            )
        t2 = timeit.default_timer()
        self.timings.update({'desc_s': t_desc, 'model_s': t1 - t0, 'int_const_s': t2 - t1, 'total_s': t2 - t_all})
        return model

    def _recov_int_const(self, model, task, R_desc=None, R_d_desc=None):
        """train.py:1090-1258: c = mean(E_ref - E_pred) over the training points.  The
        reference's dataset self-diagnostics (sign / correlation / scale warnings,
        train.py:1150-1255) are kept."""
        gdml_predict = GDMLPredict(model, max_memory=self._max_memory, max_processes=self._max_processes)
        gdml_predict.set_R_desc(R_desc)
        gdml_predict.set_R_d_desc(R_d_desc)
        E_pred, _ = gdml_predict.predict()
        E_ref = np.squeeze(task['E_train'])

        # slope of the least-squares line E_ref ~ e_fact * E_pred + b and the correlation coefficient, in closed form
        # (the reference calls np.linalg.lstsq / np.corrcoef, train.py:1150-1170; on a many-core host waking the LAPACK
        # thread pool for that 1000 x 2 problem can cost more than the rest of the training run)
        dp = E_pred - (E_pred.sum() / E_pred.size)
        dr = E_ref - (E_ref.sum() / E_ref.size)
        spp, srr, spr = float((dp * dp).sum()), float((dr * dr).sum()), float((dp * dr).sum())
        e_fact = spr / spp if spp > 0 else 1.0
        corrcoef = spr / np.sqrt(spp * srr) if spp > 0 and srr > 0 else 1.0
        if np.sign(e_fact) == -1:
            self.log.warning('The provided dataset may contain gradients instead of force labels (flipped sign).')
        if corrcoef < 0.95:
            self.log.warning(
                'Potentially inconsistent energy labels detected (correlation coefficient {:.2f}).'.format(corrcoef)
            )
        if np.abs(e_fact - 1) > 1e-1:
            self.log.warning(
                'Potentially inconsistent scales in energy vs. force labels detected (factor ~{:.2f}).'.format(e_fact)
            )
        return np.sum(E_ref - E_pred) / E_ref.shape[0]  # train.py:1258

    # ------------------------------------------------------------------ kernel matrix
    def _assemble_kernel_mat_device(
        self, R_desc, R_d_desc, tril_perms_lin, sig, col_idxs=None, scale=1.0, ldk=None, out=None, rows=None
    ):
        """K (or scale*K) assembled into a new CUDA tensor of shape (3NM, ldk); only the first
        n_cols columns are meaningful.  col_idxs: None | sorted unique int array.
        rows=(m_begin, m_end): only the block rows of these training points (row-sharded
        assembly, SURVEY.md section 8e); the tensor then has (m_end - m_begin)*3N rows."""
        torch = _torch()
        # device-resident copies of the training descriptors (cached by train()) are used in place: no H2D copy
        views = getattr(self, '_dev_views', {})
        R_desc = views.get(id(R_desc), None) if id(R_desc) in views else np.ascontiguousarray(R_desc, dtype=np.float64)
        R_d_desc = views.get(id(R_d_desc), None) if id(R_d_desc) in views else np.ascontiguousarray(R_d_desc, dtype=np.float64)
        tril_perms_lin = np.ascontiguousarray(tril_perms_lin, dtype=np.int64)
        n_train, dim_d = R_d_desc.shape[:2]
        n_atoms = int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        n_perms = len(tril_perms_lin) // dim_d
        n = n_train * 3 * n_atoms
        if col_idxs is None:
            n_cols, cols = n, None
        else:
            cols = np.ascontiguousarray(col_idxs, dtype=np.int64)
            n_cols = len(cols)
        if ldk is None:
            ldk = (n_cols + 1) // 2 * 2  # even row stride keeps the DMMA GEMM on its aligned path
        m_begin, m_end = (0, n_train) if rows is None else (int(rows[0]), int(rows[1]))
        n_rows = (m_end - m_begin) * 3 * n_atoms
        if out is not None:
            K, ldk = out, out.shape[1]
            assert K.shape[0] == n_rows and ldk >= n_cols and K.is_cuda and K.dtype == torch.float64
        else:
            K = torch.empty((n_rows, ldk), dtype=torch.float64, device='cuda')
        _lib.check(
            _lib.lib().sgdml_b200_assemble_rows(
                _lib.ptr(R_desc),
                _lib.ptr(R_d_desc),
                _lib.ptr(tril_perms_lin),
                n_atoms,
                n_train,
                n_perms,
                float(sig),
                _lib.ptr(cols),
                n_cols,
                float(scale),
                m_begin,
                m_end,
                K.data_ptr(),
                ldk,
                _lib.current_stream(),
            ),
            'assemble',
        )
        return K, n_cols

    def _assemble_kernel_mat_ecstr_device(self, R_desc, R_d_desc, tril_perms_lin, sig, scale=1.0):
        """(3NM + M)-square kernel matrix with energy constraints (train.py:234-300) as a CUDA tensor
        (n_tot, ldk): force-force part by the assembly kernel, energy rows / columns by k_assemble_ecstr."""
        torch = _torch()
        R_desc = np.ascontiguousarray(R_desc, dtype=np.float64)
        R_d_desc = np.ascontiguousarray(R_d_desc, dtype=np.float64)
        tril_perms_lin = np.ascontiguousarray(tril_perms_lin, dtype=np.int64)
        n_train, dim_d = R_d_desc.shape[:2]
        n_atoms = int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        n_perms = len(tril_perms_lin) // dim_d
        n = n_train * 3 * n_atoms
        n_tot = n + n_train
        ldk = (n_tot + 1) // 2 * 2
        K = torch.zeros((n_tot, ldk), dtype=torch.float64, device='cuda')
        self._assemble_kernel_mat_device(R_desc, R_d_desc, tril_perms_lin, sig, scale=scale, out=K[:n])
        _lib.check(
            _lib.lib().sgdml_b200_assemble_ecstr(
                _lib.ptr(R_desc), _lib.ptr(R_d_desc), _lib.ptr(tril_perms_lin), n_atoms, n_train, n_perms, float(sig),
                float(scale), K.data_ptr(), ldk, _lib.current_stream(),
            ),
            'assemble_ecstr',
        )
        return K

    def _assemble_kernel_mat_ecstr_rows_device(self, R_desc, R_d_desc, tril_perms_lin, sig, col_idxs, rows=None, scale=1.0):
        """Columns col_idxs (sorted unique, in [0, 3NM + M)) of the energy-constrained kernel matrix as a CUDA tensor
        (n_rows, ldk), first len(col_idxs) columns meaningful.  Rows: the force rows of training points
        rows=(m_begin, m_end) (default: all), then their energy rows -- (m_end - m_begin)(3N + 1) rows."""
        torch = _torch()
        views = getattr(self, '_dev_views', {})
        R_desc = views.get(id(R_desc), None) if id(R_desc) in views else np.ascontiguousarray(R_desc, dtype=np.float64)
        R_d_desc = views.get(id(R_d_desc), None) if id(R_d_desc) in views else np.ascontiguousarray(R_d_desc, dtype=np.float64)
        tril_perms_lin = np.ascontiguousarray(tril_perms_lin, dtype=np.int64)
        n_train, dim_d = R_d_desc.shape[:2]
        n_atoms = int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        n_perms = len(tril_perms_lin) // dim_d
        cols = np.ascontiguousarray(col_idxs, dtype=np.int64)
        n_cols = len(cols)
        ldk = (n_cols + 1) // 2 * 2  # even row stride, as _assemble_kernel_mat_device
        m_begin, m_end = (0, n_train) if rows is None else (int(rows[0]), int(rows[1]))
        K = torch.empty(((m_end - m_begin) * (3 * n_atoms + 1), ldk), dtype=torch.float64, device='cuda')
        _lib.check(
            _lib.lib().sgdml_b200_assemble_ecstr_rows(
                _lib.ptr(R_desc), _lib.ptr(R_d_desc), _lib.ptr(tril_perms_lin), n_atoms, n_train, n_perms, float(sig),
                _lib.ptr(cols), n_cols, float(scale), m_begin, m_end, K.data_ptr(), ldk, _lib.current_stream(),
            ),
            'assemble_ecstr_rows',
        )
        return K, n_cols

    def _assemble_kernel_mat(
        self,
        R_desc,
        R_d_desc,
        tril_perms_lin,
        sig,
        desc,
        use_E_cstr=False,
        col_idxs=np.s_[:],
        alloc_extra_rows=0,
        callback=None,
    ):
        """train.py:1260-1535: returns K as a host array of shape (3NM + alloc_extra_rows, n_cols)
        in the reference's sign convention.  (The analytic path does not use this host copy.)"""
        n_train, dim_d = R_d_desc.shape[:2]
        dim_i = 3 * int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        K_n_rows = n_train * dim_i
        if use_E_cstr:  # train.py:1333-1335: M extra rows and columns
            n_tot = K_n_rows + n_train
            if isinstance(col_idxs, slice) and col_idxs == np.s_[:]:
                Kd = self._assemble_kernel_mat_ecstr_device(R_desc, R_d_desc, tril_perms_lin, sig, scale=1.0)
                K = np.empty((n_tot + alloc_extra_rows, n_tot))
                K[:n_tot, :] = Kd[:, :n_tot].cpu().numpy()
                return K
            # column subset (the Nystroem set-up, iterative.py:232-247): the engine's rows are already in the
            # reference's order [forces; energies]
            cols = np.arange(n_tot)[col_idxs] if isinstance(col_idxs, slice) else np.asarray(col_idxs, dtype=np.int64)
            assert len(cols) == len(set(cols.tolist()))  # train.py:1337
            assert np.array_equal(cols, np.sort(cols))  # train.py:1341-1345
            if len(cols) > n_tot or (len(cols) and (cols[0] < 0 or cols[-1] >= n_tot)):
                raise ValueError('Columns indexed beyond range.')  # train.py:1349-1350
            Kd, n_cols = self._assemble_kernel_mat_ecstr_rows_device(R_desc, R_d_desc, tril_perms_lin, sig, cols)
            K = np.empty((n_tot + alloc_extra_rows, n_cols))
            K[:n_tot, :] = Kd[:, :n_cols].cpu().numpy()
            return K
        if isinstance(col_idxs, slice):
            cols = np.arange(K_n_rows)[col_idxs]
            if len(cols) == K_n_rows:
                cols = None
        else:
            cols = np.asarray(col_idxs, dtype=np.int64)
            assert len(cols) == len(set(cols.tolist()))  # train.py:1337
            assert np.array_equal(cols, np.sort(cols))  # train.py:1341-1345
        if cols is not None and len(cols) > K_n_rows:
            raise ValueError('Columns indexed beyond range.')  # train.py:1349-1350
        if callback is not None:
            callback(0, 100)
        start = timeit.default_timer()
        Kd, n_cols = self._assemble_kernel_mat_device(R_desc, R_d_desc, tril_perms_lin, sig, col_idxs=cols)
        K = np.empty((K_n_rows + alloc_extra_rows, n_cols))
        K[:K_n_rows, :] = Kd[:, :n_cols].cpu().numpy()
        if callback is not None:
            dur_s = timeit.default_timer() - start
            callback(1, 1, sec_disp_str='took {:.1f} s'.format(dur_s) if dur_s >= 0.1 else '')
        return K
