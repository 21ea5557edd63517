"""``GDMLPosterior`` -- Gaussian-process uncertainties of an analytic-solver model on the device.

An sGDML model is the posterior mean of a Gaussian process.  With C = -K_ref, the matrix ``Analytic.solve`` assembles
(layout [forces (3NM); energies (M)], the energy rows standing for -E), the training columns X (the 3NM force
columns, plus the M energy columns of a ``use_E_cstr`` model) and the factor C_XX + lam I = L L^T of training, every
query geometry q has the d = 3N + 1 outputs z_q = [F_q (3N); E_q] and

    V_q     = C(z_q, X) L^-T                            (cross rows, solved against the factor)
    Sigma_q = a^2 std^2 (P_q - V_q V_q^T),  P_q = C(z_q, z_q),  E-F entries negated (the blocks are for +E),
    a^2     = |L^-1 y|^2 / n                            (maximum-likelihood signal variance; y as train() solves it)

in the model's units squared.  The mean of the same process is the model's prediction: -std C(F_q, X) alpha is
``GDMLPredict.predict``'s F and +std C(E_q, X) alpha its E - c.

The factor is assembled and factorised once, on the device, in the constructor; queries run in chunks: the query
descriptors go into the slots after the training points of one device buffer, ``sgdml_b200_assemble_ecstr_rows``
assembles the chunk's cross rows and each query's prior block, ``sgdml_b200_trsm_right_lt`` solves the cross rows and
``sgdml_b200_posterior_blocks`` forms the blocks.  DESIGN.md section 4.1.13 has the contract and the measurements.
"""

import numpy as np

from . import _lib
from .desc import Desc
from .train import GDMLTrain, labels

# device memory left free beside a chunk's buffers (the library's staging pool, workspaces and torch's own)
_CHUNK_MARGIN_BYTES = 512 * 1024**2
_ALPHA_RTOL = 1e-6


def _torch():
    import torch

    return torch


def _even(n):
    return (n + 1) // 2 * 2  # even row stride keeps the DMMA GEMM on its aligned path


class GDMLPosterior(object):
    def __init__(self, model, task, max_memory=None):
        """Assembles C_XX + lam I of `model` (trained by the analytic solver on `task`) and factorises it on the device.

        max_memory [GB] caps the device memory the factor and one chunk of queries may take (default: what is free).
        Raises ValueError for a model not trained by the analytic solver, a factor that does not fit, a task whose
        training descriptors are not the model's, and a task whose labels, sig or lam do not reproduce the model's
        coefficients (re-solved alphas off by more than 1e-6 relative); np.linalg.LinAlgError if the matrix is not
        positive definite."""
        torch = _torch()
        _lib.require_gpu()
        if str(model.get('solver_name', '')) != 'analytic':
            raise ValueError('GDMLPosterior needs a model trained by the analytic solver (solver_name %r)'
                             % (model.get('solver_name'),))
        self.n_atoms = N = int(np.asarray(model['z']).shape[0])
        self.n_train = M = int(model['R_desc'].shape[1])
        self.use_E_cstr = 'alphas_E' in model
        self.std = float(model['std'])
        self.sig = float(model['sig'])
        self.lam = float(model['lam'])
        self.tril_perms_lin = np.ascontiguousarray(model['tril_perms_lin'], dtype=np.int64)
        self.n_perms = int(np.asarray(model['perms']).shape[0])
        self.n = n = 3 * N * M + (M if self.use_E_cstr else 0)
        self.dim = 3 * N + 1
        self.desc = Desc(N)
        self.lat_and_inv = None
        if 'lattice' in model:
            lat = np.ascontiguousarray(model['lattice'], dtype=np.float64)
            self.lat_and_inv = (lat, np.ascontiguousarray(np.linalg.inv(lat)))
        self._max_memory = max_memory
        self._max_chunk = None  # caps the queries per chunk (tests)
        self._L = None

        self.ldl = _even(n)
        factor_bytes = 8 * n * self.ldl
        budget = self._budget()
        if factor_bytes + self._chunk_bytes(1) > budget:
            raise ValueError(
                'the %d x %d factor (%.2f GB) and one chunk of queries do not fit in %.2f GB of device memory; a '
                'GDMLTrain that trained this model may still hold its kernel matrix: GDMLTrain.release_buffers() '
                'frees it' % (n, n, factor_bytes / 1024**3, budget / 1024**3))

        R = np.ascontiguousarray(task['R_train'], dtype=np.float64).reshape(M, -1)
        if R.shape[1] != 3 * N:
            raise ValueError('task geometries have %d coordinates, the model %d' % (R.shape[1], 3 * N))
        lat_and_inv = None
        if 'lattice' in task:
            lat = np.ascontiguousarray(task['lattice'], dtype=np.float64)
            lat_and_inv = (lat, np.ascontiguousarray(np.linalg.inv(lat)))
        R_desc, R_d_desc = self.desc.from_R(R, lat_and_inv=lat_and_inv)
        R_desc, R_d_desc = R_desc.reshape(M, -1), R_d_desc.reshape(M, -1, 3)
        ref = np.asarray(model['R_desc'], dtype=np.float64).T
        if ref.shape != R_desc.shape or np.max(np.abs(R_desc - ref)) > 1e-12 * max(np.max(np.abs(ref)), 1e-300):
            raise ValueError("the task's training descriptors differ from the model's R_desc: not the task it was "
                             "trained on")
        y, y_std, _ = labels(task, self.use_E_cstr)

        # descriptor buffers [M training points; query slots]; the training part is written once
        self._X = torch.from_numpy(R_desc).cuda()
        self._G = torch.from_numpy(np.ascontiguousarray(R_d_desc)).cuda()

        L = _lib.lib()
        stream = _lib.current_stream()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        gt = GDMLTrain(max_memory=max_memory)
        if self.use_E_cstr:
            K = gt._assemble_kernel_mat_ecstr_device(R_desc, R_d_desc, self.tril_perms_lin, self.sig, scale=-1.0)
        else:
            K = torch.empty((n, self.ldl), dtype=torch.float64, device='cuda')
            gt._assemble_kernel_mat_device(R_desc, R_d_desc, self.tril_perms_lin, self.sig, scale=-1.0, out=K)
        ev[1].record()
        _lib.check(L.sgdml_b200_add_diag(K.data_ptr(), n, self.ldl, self.lam, stream), 'add_diag')
        try:
            _lib.check(L.sgdml_b200_potrf(K.data_ptr(), n, self.ldl, stream), 'potrf')
            ev[2].record()
            # a^2 = |L^-1 y|^2 / n; alpha-hat = -L^-T L^-1 y must be the model's coefficients
            z = torch.zeros((1, self.ldl), dtype=torch.float64, device='cuda')
            z[0, :n] = torch.from_numpy(y).cuda()
            _lib.check(L.sgdml_b200_trsm_right_lt(K.data_ptr(), n, self.ldl, z.data_ptr(), 1, self.ldl, stream),
                       'trsm_right_lt')
            zh = z[0, :n].cpu().numpy()
            x = y.copy()
            _lib.check(L.sgdml_b200_potrs(K.data_ptr(), n, self.ldl, _lib.ptr(x), 1, 1, stream), 'potrs')
            ev[3].record()
            torch.cuda.synchronize()
            del z
        except Exception:
            del K
            self._X = self._G = None
            raise
        alphas = np.asarray(model['alphas_F'], dtype=np.float64).ravel()
        if self.use_E_cstr:
            alphas = np.hstack((alphas, np.asarray(model['alphas_E'], dtype=np.float64).ravel()))
        if alphas.shape != (n,) or np.max(np.abs(-x - alphas)) > _ALPHA_RTOL * max(np.max(np.abs(alphas)), 1e-300):
            del K
            self._X = self._G = None
            raise ValueError("re-solving the task's labels does not reproduce the model's coefficients: labels, sig "
                             "or lam do not belong to this model")
        self._L = K
        # device seconds of the constructor's three phases
        self.timings = {'assemble_s': ev[0].elapsed_time(ev[1]) * 1e-3, 'factor_s': ev[1].elapsed_time(ev[2]) * 1e-3,
                        'solve_s': ev[2].elapsed_time(ev[3]) * 1e-3}
        self.amplitude = float(zh.dot(zh)) / n
        self.scale = self.amplitude * self.std**2

    # ------------------------------------------------------------------ sizing
    def _budget(self):
        free, _total = _torch().cuda.mem_get_info()
        return free if self._max_memory is None else min(free, int(self._max_memory * 1024**3))

    def _chunk_bytes(self, c):
        """Device bytes one chunk of c queries takes: cross rows and the TRSM's panel, prior and output blocks, the
        blocks' partial sums and the descriptor slots."""
        d, D = self.dim, self.desc.dim
        nT = (d + 31) // 32
        n_slices = (self.n + 4095) // 4096
        per_query = d * (_even(self.n) + 128) + 3 * d * d + n_slices * nT * (nT + 1) // 2 * 1024 + 4 * D
        return 8 * c * per_query

    def _chunk(self, B):
        """Queries per chunk: what fits in free device memory beside a margin, at most B, the private cap and the
        assembly's 65535 points."""
        per = self._chunk_bytes(1)
        c = (self._budget() - _CHUNK_MARGIN_BYTES) // per
        if self._max_memory is not None:
            c = min(c, (int(self._max_memory * 1024**3) - 8 * self.n * self.ldl) // per)
        c = min(int(c), B, 65535 - self.n_train)
        if self._max_chunk is not None:
            c = min(c, int(self._max_chunk))
        if c < 1:
            raise RuntimeError('CUDA out of memory: one query needs %.1f MB of device memory' % (per / 1024**2))
        return c

    # ------------------------------------------------------------------ queries
    def _geometries(self, R):
        """R as GDMLPredict.predict takes it ((B, 3N), (3N,), (B, N, 3); NumPy or torch float64) -> (B, 3N) host."""
        dim_i = 3 * self.n_atoms
        if hasattr(R, 'data_ptr') and not isinstance(R, np.ndarray):
            import torch

            if R.dtype != torch.float64:
                raise ValueError('torch inputs must be float64')
            R = R.detach().cpu().numpy()
        R = np.ascontiguousarray(R, dtype=np.float64)
        if R.ndim == 1:
            R = R[None, :]
        if R.size % dim_i != 0 or (R.ndim == 2 and R.shape[1] != dim_i):
            raise ValueError('R must have 3*n_atoms columns')
        return R.reshape(-1, dim_i)

    def _slots(self, c):
        """Grows the descriptor buffers to c query slots after the training points (the training part is kept)."""
        torch = _torch()
        M, D = self.n_train, self.desc.dim
        if self._X.shape[0] < M + c:
            X = torch.empty((M + c, D), dtype=torch.float64, device='cuda')
            G = torch.empty((M + c, D, 3), dtype=torch.float64, device='cuda')
            X[:M] = self._X[:M]
            G[:M] = self._G[:M]
            self._X, self._G = X, G

    def _cross_rows(self, Rc):
        """Writes the descriptors of the geometries Rc (c, 3N) into the query slots and assembles, with scale -1,
        the cross rows C(z, X) ((3N + 1) c rows: force rows q 3N + r, then the energy rows 3N c + q; row stride
        even(n)) and the prior blocks P_q = C(z_q, z_q) ((c, d, d), order [F; E]).  Returns (V, P) CUDA tensors."""
        torch = _torch()
        L = _lib.lib()
        stream = _lib.current_stream()
        N, M, D, d = self.n_atoms, self.n_train, self.desc.dim, self.dim
        c = Rc.shape[0]
        self._slots(c)
        Xq, Gq = self._X[M:M + c], self._G[M:M + c]
        if self.lat_and_inv is not None:
            rc = L.sgdml_b200_desc_from_R_pbc(_lib.ptr(Rc), c, N, _lib.ptr(self.lat_and_inv[0]),
                                              _lib.ptr(self.lat_and_inv[1]), Xq.data_ptr(), Gq.data_ptr(), stream)
        else:
            rc = L.sgdml_b200_desc_from_R(_lib.ptr(Rc), c, N, Xq.data_ptr(), Gq.data_ptr(), stream)
        _lib.check(rc, 'desc_from_R')
        n_pts = M + c  # the joint point set [training; this chunk]
        nf = 3 * N * n_pts
        cols = np.arange(3 * N * M, dtype=np.int64)
        if self.use_E_cstr:
            cols = np.hstack((cols, nf + np.arange(M, dtype=np.int64)))
        ldv = _even(self.n)
        V = torch.empty((d * c, ldv), dtype=torch.float64, device='cuda')
        args = (self._X.data_ptr(), self._G.data_ptr(), _lib.ptr(self.tril_perms_lin), N, n_pts, self.n_perms, self.sig)
        _lib.check(L.sgdml_b200_assemble_ecstr_rows(*args, _lib.ptr(cols), self.n, -1.0, M, M + c, V.data_ptr(), ldv,
                                                    stream), 'assemble_ecstr_rows')
        # every prior block by the same one-point call, so its bits do not depend on the chunk
        P = torch.empty((c, d, d), dtype=torch.float64, device='cuda')
        for q in range(c):
            own = np.hstack((np.arange(3 * N * (M + q), 3 * N * (M + q + 1), dtype=np.int64),
                             np.array([nf + M + q], dtype=np.int64)))
            _lib.check(L.sgdml_b200_assemble_ecstr_rows(*args, _lib.ptr(own), d, -1.0, M + q, M + q + 1, P[q].data_ptr(),
                                                        d, stream), 'assemble_ecstr_rows')
        return V, P

    def _solved_rows(self, Rc):
        """_cross_rows with the cross rows solved in place against the factor: V <- C(z, X) L^-T."""
        V, P = self._cross_rows(Rc)
        _lib.check(_lib.lib().sgdml_b200_trsm_right_lt(self._L.data_ptr(), self.n, self.ldl, V.data_ptr(), V.shape[0],
                                                       V.shape[1], _lib.current_stream()), 'trsm_right_lt')
        return V, P

    def predict_cov(self, R):
        """Posterior covariance blocks (B, 3N + 1, 3N + 1) float64 (NumPy) of the outputs [F (3N, the predictor's
        order); E] of each geometry, in the model's units squared.  R in the forms GDMLPredict.predict takes; torch
        inputs are read on the host.  The blocks are exactly symmetric and returned as computed (no clamping)."""
        if self._L is None:
            raise RuntimeError('GDMLPosterior has been released')
        R = self._geometries(R)
        B, d, n = R.shape[0], self.dim, self.n
        out = np.empty((B, d, d))
        if B == 0:
            return out
        c = self._chunk(B)
        for b0 in range(0, B, c):
            b1 = min(b0 + c, B)
            V, P = self._solved_rows(np.ascontiguousarray(R[b0:b1]))
            _lib.check(_lib.lib().sgdml_b200_posterior_blocks(V.data_ptr(), V.shape[1], n, b1 - b0, self.n_atoms,
                                                              P.data_ptr(), self.scale, _lib.ptr(out[b0:b1]),
                                                              _lib.current_stream()), 'posterior_blocks')
            del V, P
        return out

    def predict_std(self, R):
        """(E_std (B,), F_std (B, 3N)): square roots of the diagonals of predict_cov, negatives from rounding
        clamped to 0."""
        cov = self.predict_cov(R)
        sd = np.sqrt(np.maximum(np.diagonal(cov, axis1=1, axis2=2), 0.0))
        return sd[:, -1].copy(), sd[:, :-1].copy()

    def release(self):
        """Frees the factor and the query workspaces."""
        self._L = None
        self._X = self._G = None
