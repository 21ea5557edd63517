"""``Iterative`` -- Nystroem-preconditioned CG (reference sgdml/solvers/iterative.py:60-866) on
the H100 engine.

Same algorithm and knobs as the reference: leverage-score sampling of inducing columns
(iterative.py:353-411), the Nystroem factor B = L_inv_K_mn (iterative.py:208-351), the
preconditioner P v = (B^T B v - v)/lam (iterative.py:136-138), the matrix-free operator
K v = predict_train(alphas = v) - lam v (iterative.py:183-204), restarts with 1.2x more inducing
points when CG stalls (iterative.py:726-801) and periodic checkpoints through
`save_progr_callback` (iterative.py:675-724).

What is different: the (n x m) block K_nm never leaves HBM -- it is assembled there
(`sgdml_b200_assemble` with a column list), factorised with the engine's FP64 Cholesky / TRSM /
Gram kernels (`csrc/nystroem.cu`, `csrc/solve.cu`), and applied with two GEMV kernels per
iteration; K v is one launch sequence of the fused predictor on the cached training descriptors.
The CG loop itself runs on the device too (`sgdml_b200_pcg`, csrc/pcg.cu): vectors and scalars never leave HBM;
the host sees a residual history every few iterations for the reference's callbacks, checkpoints and restarts.
"""

import collections
import logging
import timeit

import numpy as np

from .. import _lib

CG_STEPS_HIST_LEN = 100  # moving average window of the solver-effectiveness estimate (iterative.py:48-50)
EFF_RESTART_THRESH = 0  # restart with a stronger preconditioner below this effectiveness [%] (iterative.py:51)
MAX_NUM_RESTARTS = 6  # iterative.py:53

DONE = 1
NOT_DONE = 0


def _dot(a, b):
    """Inner product of two CG vectors without the BLAS thread pool: on the 128-thread host waking the
    pool up between two GPU calls can cost more than the K.v product itself."""
    return float(np.einsum('i,i->', a, b))


def _norm(a):
    return float(np.sqrt(np.einsum('i,i->', a, a)))


class _EngineNystroemOps(object):
    """Compute side of the row-sharded Nystroem factor (dist.nystroem_factor_steps and friends) on
    the CUDA engine: every method is one C-ABI call on this rank's rows; matrices are CUDA tensors."""

    def __init__(self, solver, R_desc, R_d_desc, tril_perms_lin, sig, use_E_cstr=False):
        self.solver = solver
        self.args = (R_desc, R_d_desc, tril_perms_lin, sig)
        self.use_E_cstr = use_E_cstr

    def assemble_rows(self, lo, hi, cols):
        if self.use_E_cstr:  # force rows of [lo, hi), then their energy rows (sgdml_b200_assemble_ecstr_rows)
            X, _ = self.solver.gdml_train._assemble_kernel_mat_ecstr_rows_device(*self.args, cols, rows=(lo, hi))
            return X
        X, _ = self.solver.gdml_train._assemble_kernel_mat_device(*self.args, col_idxs=cols, rows=(lo, hi))
        return X

    def new_square(self, m):
        import torch

        return torch.zeros((m, (m + 1) // 2 * 2), dtype=torch.float64, device='cuda')

    def put_neg_rows(self, A, pos, X, local_rows, m):
        import torch

        if len(pos) == m:  # every inducing row lives here (single rank): one gather kernel
            rows = np.ascontiguousarray(local_rows, dtype=np.int64)
            _lib.check(
                _lib.lib().sgdml_b200_gather_rows_neg(X.data_ptr(), X.shape[1], m, _lib.ptr(rows), A.data_ptr(), A.shape[1], _lib.current_stream()),
                'gather_rows_neg',
            )
        elif len(pos):
            A[torch.as_tensor(pos, device=A.device), :m] = -X[torch.as_tensor(local_rows, device=A.device), :m]

    def scaled_identity(self, m, value):
        import torch

        Y = torch.zeros((m, (m + 1) // 2 * 2), dtype=torch.float64, device='cuda')
        Y[:, :m].fill_diagonal_(float(value))
        return Y

    def add_gram(self, Y, m, A):
        G = self.new_square(m)
        self.gram(Y, m, G)
        A += G  # (only the lower triangles are meaningful)

    def trace(self, A, m):
        import torch

        return float(torch.diagonal(A[:, :m]).sum())

    def potrf(self, A):
        rc = _lib.lib().sgdml_b200_potrf(A.data_ptr(), A.shape[0], A.shape[1], _lib.current_stream())
        if rc < 0:
            _lib.check(rc, 'potrf')
        return rc == 0

    def cho_factor_stable(self, A, **kw):
        return self.solver._cho_factor_stable(A, **kw)

    def trsm_right_lt(self, A, X, m):
        _lib.check(
            _lib.lib().sgdml_b200_trsm_right_lt(A.data_ptr(), m, A.shape[1], X.data_ptr(), X.shape[0], X.shape[1], _lib.current_stream()),
            'trsm',
        )

    def gram(self, X, m, A):
        _lib.check(
            _lib.lib().sgdml_b200_gram_tn(X.data_ptr(), X.shape[0], m, X.shape[1], 0.0, A.data_ptr(), A.shape[1], _lib.current_stream()),
            'gram',
        )

    def add_diag(self, A, m, value):
        _lib.check(_lib.lib().sgdml_b200_add_diag(A.data_ptr(), m, A.shape[1], float(value), _lib.current_stream()), 'add_diag')

    def row_sqnorms(self, X, m):
        out = np.empty(X.shape[0])
        _lib.check(
            _lib.lib().sgdml_b200_row_sqnorms(X.data_ptr(), X.shape[0], m, X.shape[1], _lib.ptr(out), _lib.current_stream()),
            'row_sqnorms',
        )
        return out

    def project(self, X, m, v_loc):
        import torch

        t = torch.empty(m, dtype=torch.float64, device='cuda')
        _lib.check(
            _lib.lib().sgdml_b200_nystroem_project(X.data_ptr(), X.shape[0], m, X.shape[1], _lib.ptr(v_loc), t.data_ptr(), _lib.current_stream()),
            'nystroem_project',
        )
        return t

    def expand(self, X, m, lam, t, v_loc):
        out = np.empty(X.shape[0])
        _lib.check(
            _lib.lib().sgdml_b200_nystroem_expand(
                X.data_ptr(), X.shape[0], m, X.shape[1], float(lam), t.data_ptr(), _lib.ptr(v_loc), _lib.ptr(out), _lib.current_stream()
            ),
            'nystroem_expand',
        )
        return out


class Iterative(object):
    def __init__(self, gdml_train, desc, max_memory, max_processes, use_torch, callback=None):
        self.log = logging.getLogger(__name__)
        self.gdml_train = gdml_train
        self.gdml_predict = None
        self.desc = desc
        self.callback = callback
        self._max_memory = max_memory
        self._max_processes = max_processes
        self._use_torch = use_torch
        self.timings = {}

    def _world(self):
        """(rank, world) this solve is spread over: torch.distributed's, if the trainer was told that EVERY rank runs
        the training (`GDMLTrain.distributed = True`); (0, 1) otherwise -- e.g. rank 0 training alone while the other
        ranks wait for the coefficients, in which case no collective may be issued from here."""
        from .. import dist as sdist

        if not getattr(self.gdml_train, 'distributed', False):
            return 0, 1
        return sdist.world_info()

    # ------------------------------------------------------------------ preconditioner
    def _cho_factor_stable(self, M, pre_reg=False, eps_mag_max=1):
        """iterative.py:414-471: factorises the (m x m) CUDA tensor M in place, adding more and more
        jitter to the diagonal until it is positive definite.  Returns True, or False if even
        10**eps_mag_max did not help (callers with eps_mag_max < 1 fall back, iterative.py:312-322)."""
        import torch

        L = _lib.lib()
        m = M.shape[0]
        eps = np.finfo(float).eps
        eps_mag = int(np.floor(np.log10(eps)))
        stream = _lib.current_stream()
        if pre_reg:
            _lib.check(L.sgdml_b200_add_diag(M.data_ptr(), m, M.shape[1], float(eps), stream), 'add_diag')
            eps_mag += 1
        backup = M.clone()  # potrf overwrites its input; the reference retries from the same matrix
        for reg in 10.0 ** np.arange(eps_mag, eps_mag_max + 1):
            rc = L.sgdml_b200_potrf(M.data_ptr(), m, M.shape[1], stream)
            if rc == 0:
                return True
            if rc < 0:
                _lib.check(rc, 'potrf')
            self.log.debug('Cholesky solver needs more aggressive regularization (adding {} to diagonal)'.format(reg))
            _lib.check(L.sgdml_b200_add_diag(backup.data_ptr(), m, backup.shape[1], float(reg), stream), 'add_diag')
            M.copy_(backup)
        return False

    def _nystroem_cholesky_factor(self, R_desc, R_d_desc, tril_perms_lin, sig, lam, use_E_cstr, col_idxs, callback=None):
        """iterative.py:208-351.  Returns X = B^T as a CUDA tensor (n, ldx) whose first m columns are
        meaningful (B = L_inv_K_mn is X[:, :m].T), and m.  Single-rank form of
        dist.nystroem_factor_steps (the same steps, no exchange)."""
        from .. import dist as sdist

        n_train, dim_d = R_d_desc.shape[:2]
        dim_i = 3 * int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        cols = np.ascontiguousarray(col_idxs, dtype=np.int64)
        ops = _EngineNystroemOps(self, R_desc, R_d_desc, tril_perms_lin, sig, use_E_cstr=use_E_cstr)
        X, _, _ = sdist.run_steps_virtual(
            [sdist.nystroem_factor_steps(ops, 0, 1, n_train, dim_i, cols, lam, use_E_cstr=use_E_cstr)]
        )[0]
        return X, len(cols)

    def _shard_precon(self, n_train):
        """Row-shard the Nystroem factor over the ranks (SURVEY.md section 8e) whenever there are
        several ranks and every rank gets at least one training point."""
        rank, world = self._world()
        return world > 1 and n_train >= world

    def _init_precon_operator_sharded(self, task, R_desc, R_d_desc, tril_perms_lin, inducing_pts_idxs):
        """Row-sharded form of _init_precon_operator: every rank assembles, factorises and applies only
        the rows of its own training points; (m x m) all-reduces during the set-up, one m-vector
        all-reduce and one n-vector all-gather per application."""
        from .. import dist as sdist

        rank, world = self._world()
        lam = float(task['lam'])
        n_train = R_desc.shape[0]
        dim_i = 3 * task['R_train'].shape[1]
        m = len(inducing_pts_idxs)
        ecstr = bool(task['use_E_cstr'])
        ops = _EngineNystroemOps(self, R_desc, R_d_desc, tril_perms_lin, task['sig'], use_E_cstr=ecstr)
        X, lo, hi = sdist.run_steps(
            sdist.nystroem_factor_steps(ops, rank, world, n_train, dim_i, inducing_pts_idxs, lam, use_E_cstr=ecstr), n_train
        )
        lev_scores = sdist.run_steps(sdist.lev_scores_steps(ops, X, m, dim_i, use_E_cstr=ecstr), n_train)

        def _P_vec(v):
            return sdist.run_steps(sdist.precon_apply_steps(ops, X, m, lam, v, lo, hi, dim_i, use_E_cstr=ecstr), n_train)

        _P_vec.keepalive = X
        _P_vec.factor = (X, m, lo, hi)  # the device PCG applies the factor itself (sgdml_b200_pcg)
        return _P_vec, lev_scores

    def _init_precon_operator(self, task, R_desc, R_d_desc, tril_perms_lin, inducing_pts_idxs, callback=None):
        """iterative.py:83-142 -> (P_vec, lev_scores)."""
        if self._shard_precon(R_desc.shape[0]):
            return self._init_precon_operator_sharded(task, R_desc, R_d_desc, tril_perms_lin, inducing_pts_idxs)
        lam = float(task['lam'])
        X, m = self._nystroem_cholesky_factor(
            R_desc, R_d_desc, tril_perms_lin, task['sig'], lam, task['use_E_cstr'], inducing_pts_idxs, callback=callback
        )
        n, ldx = X.shape
        L = _lib.lib()
        lev_scores = np.empty(n)
        _lib.check(L.sgdml_b200_row_sqnorms(X.data_ptr(), n, m, ldx, _lib.ptr(lev_scores), _lib.current_stream()), 'row_sqnorms')

        def _P_vec(v):
            v = np.ascontiguousarray(v, dtype=np.float64)
            out = np.empty(n)
            _lib.check(
                L.sgdml_b200_nystroem_apply(X.data_ptr(), n, m, ldx, lam, _lib.ptr(v), _lib.ptr(out), _lib.current_stream()),
                'nystroem_apply',
            )
            return out

        _P_vec.keepalive = X
        _P_vec.factor = (X, m, 0, R_desc.shape[0])
        return _P_vec, lev_scores

    def _init_kernel_operator(self, task, R_desc, R_d_desc, tril_perms_lin, lam, n, callback=None):
        """iterative.py:144-206: K v = predict_train(alphas = v, std = 1) - lam v.  With energy constraints
        v = [v_F; v_E] and K v = [F; -E] of the predictor with alphas_F = v_F, alphas_E = v_E."""
        from ..predict import GDMLPredict

        n_train = R_desc.shape[0]
        ecstr = bool(task['use_E_cstr'])
        v_F = np.zeros(n - n_train) if ecstr else np.zeros(n)
        v_E = np.zeros(n_train) if ecstr else None
        model = self.gdml_train.create_model(task, 'cg', R_desc, R_d_desc, tril_perms_lin, 1.0, v_F, alphas_E=v_E)
        self.gdml_predict = GDMLPredict(model, max_memory=self._max_memory, max_processes=self._max_processes)
        # K.v on the int8 tensor cores (wgmma) for large descriptors (5 exact int8 slices: forces within 1.3e-10 of the FP64
        # contractions, CG tolerance 1e-4; 1.43x the FP64 contractions' throughput at BASELINE config 3 on an H100 at 400 W);
        # SGDML_B200_OZAKI_PREDICT_SLICES (0 = FP64) overrides
        import os

        if 'SGDML_B200_OZAKI_PREDICT_SLICES' not in os.environ:
            self.gdml_predict.set_contraction_slices(5)
        self.gdml_predict.set_R_desc(R_desc)
        self.gdml_predict.set_R_d_desc(R_d_desc)

        from .. import dist as sdist

        rank, world = self._world()

        def _K_vec(v):
            v = np.ascontiguousarray(v, dtype=np.float64)
            if ecstr:
                n_f = v.size - n_train
                self.gdml_predict.set_alphas(v[:n_f], alphas_E=v[n_f:])

                def rows(lo, hi):  # [F | E] of training points [lo, hi), raw sums
                    FE = np.empty((hi - lo, 3 * self.gdml_predict.n_atoms + 1))
                    E = np.empty(hi - lo)
                    FE[:, :-1] = self.gdml_predict.kmatvec_train(lo, hi, E_out=E)
                    FE[:, -1] = E
                    return FE

                FE = sdist.kmatvec_sharded(rows, n_train) if world > 1 else rows(0, n_train)
                pred = np.concatenate([FE[:, :-1].ravel(), -FE[:, -1]])  # iterative.py:196-198
                pred -= lam * v
                return pred
            self.gdml_predict.set_alphas(v)
            if world > 1:
                # SURVEY 8e: output rows (training points) sharded over the ranks, alphas replicated, one
                # all-gather of 3N*M/G doubles per application; every rank runs the same CG on replicated vectors
                pred = sdist.kmatvec_sharded(lambda lo, hi: self.gdml_predict.kmatvec_train(lo, hi), n_train).ravel()
            else:
                pred = self.gdml_predict.kmatvec_train().ravel()
            pred -= lam * v
            return pred

        return _K_vec

    def _lev_scores(self, R_desc, R_d_desc, tril_perms_lin, sig, lam, use_E_cstr, n_inducing_pts, callback=None):
        """iterative.py:353-399: leverage scores from a random subset of <= 10 points' worth of columns."""
        n_train, dim_d = R_d_desc.shape[:2]
        dim_i = 3 * int((1 + np.sqrt(8 * dim_d + 1)) / 2)
        dim_m = dim_i * min(n_inducing_pts, 10)
        # columns of the (3NM + M)-square system with energy constraints (iterative.py:372-379)
        lev_approx_idxs = np.sort(np.random.choice(n_train * dim_i + (n_train if use_E_cstr else 0), dim_m, replace=False))
        if self._shard_precon(n_train):
            from .. import dist as sdist

            rank, world = self._world()
            lev_approx_idxs = self._bcast_idxs(lev_approx_idxs)  # one draw (rank 0's) for the shared factor
            ops = _EngineNystroemOps(self, R_desc, R_d_desc, tril_perms_lin, sig, use_E_cstr=use_E_cstr)
            X, lo, hi = sdist.run_steps(
                sdist.nystroem_factor_steps(ops, rank, world, n_train, dim_i, lev_approx_idxs, lam, use_E_cstr=use_E_cstr),
                n_train,
            )
            return sdist.run_steps(sdist.lev_scores_steps(ops, X, len(lev_approx_idxs), dim_i, use_E_cstr=use_E_cstr), n_train)
        X, m = self._nystroem_cholesky_factor(R_desc, R_d_desc, tril_perms_lin, sig, lam, use_E_cstr, lev_approx_idxs)
        lev = np.empty(X.shape[0])
        _lib.check(
            _lib.lib().sgdml_b200_row_sqnorms(X.data_ptr(), X.shape[0], m, X.shape[1], _lib.ptr(lev), _lib.current_stream()),
            'row_sqnorms',
        )
        return lev

    def inducing_pts_from_lev_scores(self, lev_scores, N):
        """iterative.py:401-411."""
        idxs = np.random.choice(np.arange(lev_scores.size), N, replace=False, p=lev_scores / lev_scores.sum())
        return np.sort(idxs)

    # ------------------------------------------------------------------ solve
    def solve(self, task, R_desc, R_d_desc, tril_perms_lin, y, y_std, tol=1e-4, save_progr_callback=None):
        """iterative.py:473-825 -> (alphas, tol, num_iters, resid, train_rmse, inducing_pts_idxs, is_conv)."""
        n_train, n_atoms = task['R_train'].shape[:2]
        dim_i = 3 * n_atoms
        sig, lam = task['sig'], float(task['lam'])

        alphas0_F = task['alphas0_F'] if 'alphas0_F' in task else None
        alphas0_E = task['alphas0_E'] if 'alphas0_E' in task else None
        ecstr = bool(task['use_E_cstr'])
        num_iters0 = int(task['solver_iters']) if 'solver_iters' in task else 0

        max_memory_bytes = self._max_memory * 1024**3
        n_inducing_pts = min(n_train, Iterative.max_n_inducing_pts(n_train, n_atoms, max_memory_bytes))
        n_inducing_pts = max(n_inducing_pts, 1)
        n_inducing_pts_init = len(task['inducing_pts_idxs']) // dim_i if 'inducing_pts_idxs' in task else None

        t_start = timeit.default_timer()
        lev_scores = None
        if n_inducing_pts_init is not None and n_inducing_pts_init == n_inducing_pts:
            inducing_pts_idxs = np.asarray(task['inducing_pts_idxs'])  # reuse old inducing points
        else:
            lev_scores = self._lev_scores(R_desc, R_d_desc, tril_perms_lin, sig, lam, task['use_E_cstr'], n_inducing_pts)
            inducing_pts_idxs = self.inducing_pts_from_lev_scores(lev_scores, n_inducing_pts * dim_i)
            self.timings['lev_scores_s'] = timeit.default_timer() - t_start

        inducing_pts_idxs = self._bcast_idxs(inducing_pts_idxs)
        P_vec, lev_scores = self._init_precon_operator(task, R_desc, R_d_desc, tril_perms_lin, inducing_pts_idxs)
        self.timings['precon_s'] = timeit.default_timer() - t_start

        n = lev_scores.size
        self._init_kernel_operator(task, R_desc, R_d_desc, tril_perms_lin, lam, n)  # -> self.gdml_predict

        y = np.ascontiguousarray(y, dtype=np.float64)
        norm_y = _norm(y)
        x0 = None
        if alphas0_F is not None:  # iterative.py:608-613: x0 = -[alphas0_F; alphas0_E]
            x0 = -np.asarray(alphas0_F, dtype=np.float64).ravel()
            if ecstr:
                a0_E = np.zeros(n_train) if alphas0_E is None else np.asarray(alphas0_E, dtype=np.float64).ravel()
                x0 = np.concatenate([x0, -a0_E])
        maxiter = 3 * n_atoms * n_train * 10  # iterative.py:746-749

        state = {
            'num_iters': num_iters0,
            'resid': None,
            'steps_hist': collections.deque(maxlen=CG_STEPS_HIST_LEN),
            'restart': False,
            'last_ckpt': timeit.default_timer(),
            'x_dev': None,
        }

        def on_progress(resids):
            """Host side of the solve, once per residual-history read-back: solver effectiveness and restart
            decision (iterative.py:640-653, 726-735), progress display, periodic checkpoints (iterative.py:675-724)."""
            for resid in resids:
                old_resid = state['resid']
                state['resid'] = resid
                state['num_iters'] += 1
                state['steps_hist'].append(resid - old_resid)
                arr = np.array(state['steps_hist'])
                tot = np.abs(arr).sum()
                ratio = (-arr.clip(max=0).sum() / tot) if tot > 0 else 1
                eff = (int(100 * ratio) - 50) * 2
                if self.callback is not None:
                    self.callback(
                        NOT_DONE,
                        disp_str='Training error (RMSE): forces {:.4f}'.format(resid / np.sqrt(len(y))),
                        sec_disp_str='{:d} iter, k={:d}'.format(state['num_iters'], n_inducing_pts),
                    )
                if len(state['steps_hist']) == CG_STEPS_HIST_LEN and eff <= EFF_RESTART_THRESH and n_inducing_pts < n_train:
                    state['restart'] = True  # iterative.py:726-735
                    return 1
            now = timeit.default_timer()
            if save_progr_callback is not None and now - state['last_ckpt'] > 120.0:
                state['last_ckpt'] = now
                xk = state['x_dev'].cpu().numpy()
                save_progr_callback(
                    self._checkpoint_model(
                        task, R_desc, R_d_desc, tril_perms_lin, y_std, xk, tol, state['num_iters'], state['resid'], norm_y, inducing_pts_idxs
                    )
                )
            return 0

        num_restarts = 0
        is_conv = False
        t_cg = timeit.default_timer()
        x = x0
        while True:  # restart loop (iterative.py:737-801)
            state['restart'] = False
            x, resid = self._pcg_device(P_vec.factor, lam, y, x, tol * norm_y, maxiter, dim_i, on_progress, state, ecstr=ecstr)
            if not state['restart']:
                is_conv = resid <= tol * norm_y
                break
            num_restarts += 1
            state['steps_hist'].clear()
            if num_restarts == MAX_NUM_RESTARTS:
                is_conv = False
                break
            n_inducing_pts = min(int(np.ceil(1.2 * n_inducing_pts)), n_train)
            inducing_pts_idxs = self._bcast_idxs(self.inducing_pts_from_lev_scores(lev_scores, n_inducing_pts * dim_i))
            del P_vec
            P_vec, lev_scores = self._init_precon_operator(task, R_desc, R_d_desc, tril_perms_lin, inducing_pts_idxs)
        num_iters = state['num_iters']

        self.timings['cg_s'] = timeit.default_timer() - t_cg
        self.timings['iters'] = num_iters - num_iters0
        alphas = -x
        train_rmse = resid / np.sqrt(len(y))
        if self.callback is not None:
            self.callback(
                DONE,
                disp_str='Training on {:,} points'.format(n_train) + ('' if is_conv else ' (NOT CONVERGED)'),
                sec_disp_str='{:d} iterations'.format(num_iters),
            )
        return alphas, tol, num_iters, resid, train_rmse, inducing_pts_idxs, is_conv

    def _pcg_device(self, factor, lam, y, x0, tol_abs, maxiter, dim_i, on_progress, state, check_every=25, ecstr=False):
        """One run of the device-resident PCG (`sgdml_b200_pcg`, csrc/pcg.cu): every CG vector stays in HBM, the
        host gets the residual history every <= check_every iterations.  With several ranks the K.v rows and the
        Nystroem factor rows are those of this rank's training points and the three exchanges per iteration run
        as torch.distributed collectives on views of the device workspace (dist.exchange_on_workspace).
        ecstr: the (3NM + M)-square energy-constrained system (`sgdml_b200_pcg_ecstr`), vectors [forces; energies];
        the energy tails of K.v and P.v are exchanged separately (op 2)."""
        import ctypes

        import torch

        from .. import dist as sdist

        L = _lib.lib()
        X, m, lo, hi = factor
        rank, world = self._world()
        n_train = self.gdml_predict.n_train
        n = n_train * dim_i + (n_train if ecstr else 0)
        if world == 1:
            lo, hi = 0, n_train
        n_rows_loc = (hi - lo) * (dim_i + 1 if ecstr else dim_i)
        ws_fn = L.sgdml_b200_pcg_ecstr_workspace_doubles if ecstr else L.sgdml_b200_pcg_workspace_doubles
        ws_doubles = int(ws_fn(n, n_rows_loc, m, check_every))
        ws = torch.empty(ws_doubles, dtype=torch.float64, device='cuda')
        state['x_dev'] = ws[:n]  # the solution vector is the first slot of the workspace (csrc/pcg.cu)
        if state['resid'] is None:
            state['resid'] = float(_norm(y)) if x0 is None else None

        def _exchange(_ctx, op, buf, count):
            try:
                off = (int(buf) - ws.data_ptr()) // 8
                sdist.exchange_on_workspace(ws, off, int(count), int(op), n_train, dim_i)
                return 0
            except Exception as e:  # noqa: BLE001 -- must not propagate through the C frame
                self.log.error('exchange failed: %r' % (e,))
                return 1

        first = {'pending': x0 is not None}

        def _progress(_ctx, iters_done, hist, n_new):
            try:
                resids = [hist[i] for i in range(n_new)]
                if first['pending']:  # warm start: the step history starts from the first measured residual
                    first['pending'] = False
                    if state['resid'] is None:
                        state['resid'] = resids[0]
                return int(on_progress(resids))
            except Exception as e:  # noqa: BLE001
                self.log.error('progress callback failed: %r' % (e,))
                state['error'] = e
                return 1

        exch = _lib.EXCHANGE_FN(_exchange) if world > 1 else ctypes.cast(None, _lib.EXCHANGE_FN)
        prog = _lib.PROGRESS_FN(_progress)
        x = np.zeros(n) if x0 is None else np.ascontiguousarray(x0, dtype=np.float64)
        iters, resid = ctypes.c_int64(0), ctypes.c_double(0.0)
        pcg = L.sgdml_b200_pcg_ecstr if ecstr else L.sgdml_b200_pcg
        _lib.check(
            pcg(
                self.gdml_predict._handle, lo, hi, X.data_ptr() if m > 0 else None, m, X.shape[1] if m > 0 else 0,
                float(lam), _lib.ptr(y), _lib.ptr(x), 1 if x0 is None else 0, float(tol_abs), int(maxiter),
                int(check_every), ws.data_ptr(), ws_doubles, exch, None, prog, None,
                ctypes.byref(iters), ctypes.byref(resid), _lib.current_stream(),
            ),
            'pcg',
        )
        if 'error' in state:
            raise state.pop('error')
        state['x_dev'] = None
        return x, float(resid.value)

    def _bcast_idxs(self, idxs):
        """The leverage-score sampling is random (iterative.py:404-409): with several ranks, rank 0's draw is
        broadcast so that every rank builds the same preconditioner."""
        from .. import dist as sdist

        rank, world = self._world()
        if world == 1:
            return idxs
        import torch
        import torch.distributed as dist

        dev = sdist._device_for_backend()
        t = torch.from_numpy(np.ascontiguousarray(idxs, dtype=np.int64)).to(dev)
        dist.broadcast(t, src=0)
        return t.cpu().numpy()

    def _checkpoint_model(self, task, R_desc, R_d_desc, tril_perms_lin, y_std, xk, tol, num_iters, resid, norm_y, idxs):
        """iterative.py:685-724: the current iterate as a model (alphas_F and, with energy constraints, alphas_E)."""
        alphas_F, alphas_E = -xk, None
        if task['use_E_cstr']:
            n_train = R_desc.shape[0]
            alphas_F, alphas_E = -xk[:-n_train], -xk[-n_train:]
        model = self.gdml_train.create_model(task, 'cg', R_desc, R_d_desc, tril_perms_lin, y_std, alphas_F, alphas_E=alphas_E)
        model.update(
            {
                'solver_tol': tol,
                'solver_iters': num_iters,
                'solver_resid': resid,
                'norm_y_train': norm_y,
                'inducing_pts_idxs': idxs,
            }
        )
        model['c'] = 0
        if 'E_train' in task:
            self.gdml_predict.set_alphas(alphas_F, alphas_E=alphas_E)
            E_pred = self.gdml_predict.predict()[0]  # std = 1, c = 0 model
            model['c'] = np.mean(np.squeeze(task['E_train']) - E_pred * y_std)
        return model

    # ------------------------------------------------------------------ memory heuristics
    @staticmethod
    def max_n_inducing_pts(n_train, n_atoms, max_memory_bytes):
        """iterative.py:826-843 (same formula, device memory instead of host memory)."""
        SQUARE_FACT, LINEAR_FACT = 5, 4
        to_dof = (3 * n_atoms) ** 2 * 8
        sq_factor = LINEAR_FACT * n_train * to_dof
        ny_factor = SQUARE_FACT * to_dof
        n_inducing_pts = (np.sqrt(sq_factor**2 + 4.0 * ny_factor * max_memory_bytes) - sq_factor) / (2 * ny_factor)
        return min(int(n_inducing_pts), n_train)

    @staticmethod
    def est_memory_requirement(n_train, n_inducing_pts, n_atoms):
        """iterative.py:845-866."""
        SQUARE_FACT, LINEAR_FACT = 5, 4
        est_bytes = LINEAR_FACT * n_train * n_inducing_pts * (3 * n_atoms) ** 2 * 8
        est_bytes += SQUARE_FACT * n_inducing_pts * n_inducing_pts * (3 * n_atoms) ** 2 * 8
        return est_bytes
