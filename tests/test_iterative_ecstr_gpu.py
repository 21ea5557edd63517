"""Nystroem-preconditioned CG with energy constraints on the engine (H100): sgdml_b200_assemble_ecstr_rows,
sgdml_b200_pcg_ecstr and GDMLTrain.train(use_E_cstr) on a system routed to the iterative solver, against the oracle
and the reference's run frozen in tests/golden/cg_ecstr_n9_m40.npz."""

import ctypes

import numpy as np
import pytest

import ecstr_oracle as eoracle
from conftest import rel_err
from test_iterative import _np_pcg
from test_iterative_ecstr import iters_close, setup_ecstr, sharded_cols

from oracle import assemble as oassemble
from oracle import desc as odesc
from oracle import iterative as oiter

pytestmark = pytest.mark.gpu


def _assemble_rows(x, gd, lin, sig, cols, lo, hi, ldk, scale=1.0):
    import torch

    from sgdml_b200 import _lib

    M, D = x.shape
    N = odesc.n_atoms_from_dim(D)
    cols = np.ascontiguousarray(cols, dtype=np.int64)
    # the oracle's descriptors are views: contiguous copies that outlive the call
    x, gd, lin = np.ascontiguousarray(x), np.ascontiguousarray(gd), np.ascontiguousarray(lin, dtype=np.int64)
    K = torch.full(((hi - lo) * (3 * N + 1), ldk), float('nan'), dtype=torch.float64, device='cuda')
    _lib.check(
        _lib.lib().sgdml_b200_assemble_ecstr_rows(
            _lib.ptr(x), _lib.ptr(gd), _lib.ptr(lin), N, M, len(lin) // D, float(sig), _lib.ptr(cols), len(cols), float(scale), lo, hi, K.data_ptr(), ldk, _lib.current_stream(),
        ),
        'assemble_ecstr_rows',
    )
    return K.cpu().numpy()


def _rows(lo, hi, dim_i, M):
    return np.concatenate([np.arange(lo * dim_i, hi * dim_i), M * dim_i + np.arange(lo, hi)])


def _check_assembly(x, gd, lin, sig, K_full, cols, lo, hi, pad):
    M = x.shape[0]
    dim_i = 3 * odesc.n_atoms_from_dim(x.shape[1])
    K = _assemble_rows(x, gd, lin, sig, cols, lo, hi, len(cols) + pad)
    ref = K_full[_rows(lo, hi, dim_i, M)][:, cols]
    assert rel_err(K[:, : len(cols)], ref) < 1e-12
    assert np.isnan(K[:, len(cols) :]).all()  # padding columns are not written


def test_assemble_ecstr_rows_matches_oracle():
    g, task, N, M, x, gd, lin = setup_ecstr()
    sig = int(g['sig'])
    K_full = oassemble.assemble_E_cstr(x, gd, lin, sig)
    n_f, n_t = 3 * N * M, 3 * N * M + M
    rng = np.random.default_rng(3)
    col_lists = {
        'force': np.sort(rng.choice(n_f, 50, replace=False)),
        'energy': np.sort(rng.choice(np.arange(n_f, n_t), 7, replace=False)),
        'mixed': np.union1d(np.sort(rng.choice(n_f, 40, replace=False)), [n_f + 3, n_f + 20, n_t - 1]),
        'last': np.array([n_t - 1]),
        'fixture': g['inducing_pts_idxs'],
    }
    for cols in col_lists.values():
        for lo, hi in ((0, M), (13, 29), (M - 1, M)):
            _check_assembly(x, gd, lin, sig, K_full, cols, lo, hi, pad=3)
    # against the reference's own columns
    K = _assemble_rows(x, gd, lin, sig, g['inducing_pts_idxs'], 0, M, len(g['inducing_pts_idxs']) + 1)
    assert rel_err(K[:, :-1], g['K_nm']) < 1e-12


def test_assemble_ecstr_rows_large_descriptor():
    """N = 24 (D = 276 > 256): the force prefix goes through the large-descriptor assembly kernels."""
    from sgdml_b200 import synth

    N, M, sig = 24, 6, 30
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, sig)
    x, gd = odesc.from_R(task['R_train'].reshape(M, -1))
    lin = odesc.tril_perms_lin(perms)
    K_full = oassemble.assemble_E_cstr(x, gd, lin, sig)
    n_f = 3 * N * M
    cols = np.union1d(np.sort(np.random.default_rng(1).choice(n_f, 60, replace=False)), [n_f, n_f + 4])
    for lo, hi in ((0, M), (2, 5)):
        _check_assembly(x, gd, lin, sig, K_full, cols, lo, hi, pad=2)


def test_assemble_ecstr_rows_rejects_bad_input():
    from sgdml_b200 import _lib

    g, task, N, M, x, gd, lin = setup_ecstr()
    n_t = 3 * N * M + M
    for cols, lo, hi in (([5, 3], 0, M), ([0, n_t], 0, M), ([1, 1], 0, M), ([2], 3, 3), ([2], 0, M + 1)):
        with pytest.raises(_lib.EngineError):
            _assemble_rows(x, gd, lin, int(g['sig']), cols, lo, hi, 4)


def _engine_setup(g, task, N, M):
    import sgdml_b200
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    d = Desc(N)
    xe, gde = d.from_R(task['R_train'].reshape(M, -1))
    t = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    return Iterative(t, d, float(g['max_memory_gb']), None, False), xe, gde


def test_engine_ecstr_preconditioner_and_kernel_operator():
    from test_iterative_ecstr import model_like_ecstr

    g, task, N, M, x, gd, lin = setup_ecstr()
    it, xe, gde = _engine_setup(g, task, N, M)
    P, lev = it._init_precon_operator(task, xe, gde, lin, g['inducing_pts_idxs'])
    assert lev.size == 3 * N * M + M
    assert rel_err(lev, g['lev_scores']) < 1e-6
    assert rel_err(P(g['v']), g['Pv']) < 1e-5
    n = 3 * N * M + M
    K = it._init_kernel_operator(task, xe, gde, lin, float(g['lam']), n)
    Kref = eoracle.kernel_op_ecstr(model_like_ecstr(g, task, x, gd, np.zeros(n)), x, gd, float(g['lam']))
    assert rel_err(K(g['v']), Kref(g['v'])) < 1e-10


@pytest.mark.parametrize('world', [2, 3])
def test_engine_ecstr_sharded_preconditioner_virtual_ranks(world):
    from sgdml_b200 import dist as sdist
    from sgdml_b200.solvers.iterative import _EngineNystroemOps

    g, task, N, M, x, gd, lin = setup_ecstr()
    it, xe, gde = _engine_setup(g, task, N, M)
    lam, dim_i = float(g['lam']), 3 * N
    for cols, lev_ref, Pv_ref in (
        (g['inducing_pts_idxs'], g['lev_scores'], g['Pv']),
        (sharded_cols(g), None, None),  # an energy column on the last rank
    ):
        if lev_ref is None:
            B = eoracle.nystroem_factor_ecstr(x, gd, lin, int(g['sig']), lam, cols)
            lev_ref, Pv_ref = np.einsum('ij,ij->j', B, B), oiter.precon(B, lam)(g['v'])
        ops = [_EngineNystroemOps(it, xe, gde, lin, task['sig'], use_E_cstr=True) for _ in range(world)]
        facs = sdist.run_steps_virtual(
            [sdist.nystroem_factor_steps(ops[r], r, world, M, dim_i, cols, lam, use_E_cstr=True) for r in range(world)]
        )
        assert sum(f[0].shape[0] for f in facs) == M * (dim_i + 1)
        levs = sdist.run_steps_virtual([sdist.lev_scores_steps(ops[r], facs[r][0], len(cols), dim_i, use_E_cstr=True) for r in range(world)])
        Pvs = sdist.run_steps_virtual(
            [sdist.precon_apply_steps(ops[r], facs[r][0], len(cols), lam, g['v'], facs[r][1], facs[r][2], dim_i, use_E_cstr=True) for r in range(world)]
        )
        for r in range(world):
            assert rel_err(levs[r], lev_ref) < 1e-6
            assert rel_err(Pvs[r], Pv_ref) < 1e-5
            assert np.array_equal(Pvs[r], Pvs[0])


def _pcg_ecstr_call(pred, X, m, lam, y, x0, max_iters, check_every=5, progress=None):
    import torch

    from sgdml_b200 import _lib

    L = _lib.lib()
    n = y.size
    wsd = int(L.sgdml_b200_pcg_ecstr_workspace_doubles(n, n, m, check_every))
    assert wsd > int(L.sgdml_b200_pcg_workspace_doubles(n, n, m, check_every))
    ws = torch.empty(wsd, dtype=torch.float64, device='cuda')
    x = np.zeros(n) if x0 is None else np.array(x0, dtype=np.float64)
    iters, resid = ctypes.c_int64(0), ctypes.c_double(0.0)
    prog = _lib.PROGRESS_FN(progress) if progress is not None else ctypes.cast(None, _lib.PROGRESS_FN)
    _lib.check(
        L.sgdml_b200_pcg_ecstr(
            pred._handle, 0, pred.n_train, X.data_ptr() if m else None, m, X.shape[1] if m else 0, float(lam), _lib.ptr(y),
            _lib.ptr(x), 1 if x0 is None else 0, 0.0, int(max_iters), int(check_every), ws.data_ptr(), wsd,
            ctypes.cast(None, _lib.EXCHANGE_FN), None, prog, None, ctypes.byref(iters), ctypes.byref(resid), _lib.current_stream(),
        ),
        'pcg_ecstr',
    )
    return x, int(iters.value), float(resid.value)


def _check_pcg(it, task, x, gd, lin, sig, lam, y, cols, precon, warm, n_it=12):
    K = oassemble.assemble_E_cstr(x, gd, lin, sig)
    n = K.shape[0]
    A = -K + lam * np.eye(n)
    if precon:
        P, _ = it._init_precon_operator(task, x, gd, lin, cols)
        X, m = P.factor[0], P.factor[1]
        Xh = X[:, :m].cpu().numpy()
        Pinv = lambda v: (Xh @ (Xh.T @ v) - v) / lam  # noqa: E731
    else:
        X, m = None, 0
        Pinv = lambda v: v.copy()  # noqa: E731
    x0 = 0.01 * np.random.default_rng(5).standard_normal(n) if warm else None
    x_ref, hist_ref = _np_pcg(A, Pinv, y, x0, n_it)
    seen = []

    def progress(_ctx, iters_done, hist, n_new):
        seen.extend(hist[i] for i in range(n_new))
        return 0

    xs, iters, resid = _pcg_ecstr_call(it.gdml_predict, X, m, lam, y, x0, n_it, progress=progress)
    assert iters == n_it and len(seen) == n_it
    # the first iterations agree to rounding.  Without the preconditioner the residual of the fixture's system jumps
    # five-fold around iterations 6-8 (a near-breakdown of CG on a system of condition ~1e11): there the residual
    # norms of two runs that differ by rounding differ by up to 84 % (measured on an H100), and both runs recover, so
    # the rest of the history is compared from iteration 9 on, at the bound of test_pcg_c_abi_matches_numpy_cg
    assert rel_err(np.array(seen[:5]), hist_ref[:5]) < 1e-6
    assert rel_err(np.array(seen[-4:]), hist_ref[-4:]) < 1e-3
    assert rel_err(xs, x_ref) < 1e-2
    assert abs(resid - hist_ref[-1]) < 1e-3 * hist_ref[-1]


@pytest.mark.parametrize('precon', [False, True])
@pytest.mark.parametrize('warm', [False, True])
def test_pcg_ecstr_matches_numpy_cg(precon, warm):
    g, task, N, M, x, gd, lin = setup_ecstr()
    it, xe, gde = _engine_setup(g, task, N, M)
    lam = float(g['lam'])
    it._init_kernel_operator(task, xe, gde, lin, lam, 3 * N * M + M)
    _check_pcg(it, task, xe, gde, lin, int(g['sig']), lam, np.ascontiguousarray(g['y']), g['inducing_pts_idxs'], precon, warm)


def test_pcg_ecstr_large_descriptor_int8_kv():
    """N = 24 (D = 276): K.v through the GEMM-composed predictor with its default 5 int8 slices."""
    import sgdml_b200
    from sgdml_b200 import synth
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    N, M, sig = 24, 8, 30
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, sig)
    task['use_E_cstr'] = True
    lam = float(task['lam'])
    d = Desc(N)
    x, gd = d.from_R(task['R_train'].reshape(M, -1))
    lin = odesc.tril_perms_lin(perms)
    it = Iterative(sgdml_b200.GDMLTrain(max_memory=1.0), d, 1.0, None, False)
    n = 3 * N * M + M
    it._init_kernel_operator(task, x, gd, lin, lam, n)
    y = np.random.default_rng(2).standard_normal(n)
    cols = np.union1d(np.sort(np.random.default_rng(4).choice(3 * N * M, 3 * N, replace=False)), [3 * N * M + 1])
    _check_pcg(it, task, x, gd, lin, sig, lam, y, cols, precon=True, warm=False, n_it=8)


def test_engine_cg_ecstr_train_matches_reference():
    """GDMLTrain.train(use_E_cstr) routed to the iterative solver with the fixture's inducing columns; then a resume
    from a checkpoint model (alphas0_F / alphas0_E) converges in fewer iterations than the cold start."""
    import sgdml_b200

    g, task, N, M, x, gd, lin = setup_ecstr()
    task['inducing_pts_idxs'] = g['inducing_pts_idxs']
    trainer = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    from sgdml_b200.solvers import iterative as siter

    model = trainer.train(task)
    assert model['solver_name'] == 'cg' and 'alphas_E' in model and model['alphas_E'].shape == (M,)
    assert np.array_equal(model['inducing_pts_idxs'], g['inducing_pts_idxs'])
    assert model['solver_resid'] <= float(g['solver_tol']) * float(g['norm_y_train'])
    iters = int(model['solver_iters'])
    assert iters_close(iters, int(g['solver_iters_fixed_cols']))
    E, F = sgdml_b200.GDMLPredict(model).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 2e-3
    assert rel_err(E, g['E_query']) < 2e-3
    exact = sgdml_b200.GDMLTrain().train({k: v for k, v in task.items() if k != 'inducing_pts_idxs'})
    assert exact['solver_name'] == 'analytic' and 'alphas_E' in exact
    _, F_exact = sgdml_b200.GDMLPredict(exact).predict(g['R_query'])
    assert rel_err(F, F_exact) < 5e-3

    # checkpoint after a partial solve (iterative.py:675-724), then resume from it (train.py:713-717)
    orig = siter.Iterative._pcg_device

    def partial(self, factor, lam, y, x0, tol_abs, maxiter, dim_i, on_progress, state, check_every=25, ecstr=False):
        return orig(self, factor, lam, y, x0, tol_abs, min(maxiter, iters // 2), dim_i, on_progress, state, check_every, ecstr)

    siter.Iterative._pcg_device = partial
    try:
        half = trainer.train(task)
    finally:
        siter.Iterative._pcg_device = orig
    assert int(half['solver_iters']) == iters // 2 and half['solver_resid'] > model['solver_resid']
    ck = dict(task, alphas0_F=half['alphas_F'], alphas0_E=half['alphas_E'])
    resumed = trainer.train(ck)
    assert resumed['solver_resid'] <= float(g['solver_tol']) * float(g['norm_y_train'])
    assert int(resumed['solver_iters']) < iters
    _, F_res = sgdml_b200.GDMLPredict(resumed).predict(g['R_query'])
    assert rel_err(F_res, F_exact) < 5e-3


def _cg_ecstr_rank(rank, world, port, out_dir):
    import os
    import sys

    import torch
    import torch.distributed as dist

    from conftest import ROOT

    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    import sgdml_b200

    g, task, N, M, x, gd, lin = setup_ecstr()
    task['inducing_pts_idxs'] = g['inducing_pts_idxs']
    trainer = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    trainer.distributed = True
    model = trainer.train(task)
    np.savez(
        os.path.join(out_dir, 'e%d.npz' % rank), alphas_F=model['alphas_F'], alphas_E=model['alphas_E'],
        iters=model['solver_iters'], resid=model['solver_resid'], norm_y=model['norm_y_train'],
    )
    dist.barrier()
    dist.destroy_process_group()


def test_engine_cg_ecstr_two_ranks():
    import socket

    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import tempfile

    import torch.multiprocessing as mp

    import sgdml_b200

    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_cg_ecstr_rank, args=(2, port, d), nprocs=2, join=True)
        r0, r1 = dict(np.load(d + '/e0.npz')), dict(np.load(d + '/e1.npz'))
    assert np.array_equal(r0['alphas_F'], r1['alphas_F']) and np.array_equal(r0['alphas_E'], r1['alphas_E'])
    g, task, N, M, x, gd, lin = setup_ecstr()
    task['inducing_pts_idxs'] = g['inducing_pts_idxs']
    single = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb'])).train(task)
    assert float(r0['resid']) <= 1e-4 * float(r0['norm_y'])
    assert abs(int(single['solver_iters']) - int(r0['iters'])) <= max(5, 0.2 * int(r0['iters']))
    a0 = np.concatenate([r0['alphas_F'], r0['alphas_E']])
    a1 = np.concatenate([single['alphas_F'], single['alphas_E']])
    assert rel_err(a0, a1) < 2e-2
