"""Nystroem-preconditioned CG (SURVEY.md section 8 row a-S2): oracle and engine against the
reference's own iterative solve frozen in tests/golden/cg_n9_m40.npz (fixed inducing columns)."""

import numpy as np
import pytest

from conftest import load_golden, rel_err

from oracle import desc as odesc
from oracle import iterative as oiter
from oracle import predict as opredict


def _setup():
    from sgdml_b200 import synth

    g = load_golden('cg_n9_m40')
    N, M = int(g['n_atoms']), int(g['n_train'])
    task = synth.make_task(N, M, g['perms'], int(g['sig']), lam=float(g['lam']))
    R = task['R_train'].reshape(M, -1)
    return g, task, N, M, R


def _model_like(g, task, R_desc, alphas):
    N = int(g['n_atoms'])
    R = task['R_train'].reshape(R_desc.shape[0], -1)
    _, gd = odesc.from_R(R)
    return {
        'type': 'm',
        'z': task['z'],
        'R_desc': R_desc.T,
        'R_d_desc_alpha': odesc.d_desc_dot_vec(gd, alphas.reshape(-1, 3 * N)),
        'alphas_F': alphas,
        'c': float(g['c']),
        'std': float(g['std']),
        'sig': int(g['sig']),
        'lam': float(g['lam']),
        'perms': g['perms'],
        'tril_perms_lin': odesc.tril_perms_lin(g['perms']),
        'use_E': True,
    }


def test_oracle_preconditioner_and_solve():
    g, task, N, M, R = _setup()
    x, gd = odesc.from_R(R)
    lin = odesc.tril_perms_lin(g['perms'])
    B = oiter.nystroem_factor(x, gd, lin, int(g['sig']), float(g['lam']), g['inducing_pts_idxs'])
    assert rel_err(np.einsum('ij,ij->j', B, B), g['lev_scores']) < 1e-6
    assert rel_err(oiter.precon(B, float(g['lam']))(g['v']), g['Pv']) < 1e-5
    alphas, info, iters, _ = oiter.solve(
        _model_like(g, task, x, np.zeros(3 * N * M)), x, gd, lin, int(g['sig']), float(g['lam']), g['y'], g['inducing_pts_idxs']
    )
    assert info == 0
    assert abs(iters - int(g['solver_iters'])) <= max(5, 0.2 * int(g['solver_iters']))
    E, F = opredict.Predictor(_model_like(g, task, x, alphas)).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 2e-3  # both are converged to rtol 1e-4 only


@pytest.mark.gpu
def test_engine_preconditioner_matches_reference():
    import sgdml_b200
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    g, task, N, M, R = _setup()
    t = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    d = Desc(N)
    x, gd = d.from_R(R)
    lin = odesc.tril_perms_lin(g['perms'])
    it = Iterative(t, d, float(g['max_memory_gb']), None, False)
    P, lev = it._init_precon_operator(task, x, gd, lin, g['inducing_pts_idxs'])
    assert rel_err(lev, g['lev_scores']) < 1e-6
    assert rel_err(P(g['v']), g['Pv']) < 1e-5
    K = it._init_kernel_operator(task, x, gd, lin, float(g['lam']), 3 * N * M)
    Kref = oiter.kernel_op(_model_like(g, task, x, np.zeros(3 * N * M)), x, gd, float(g['lam']))
    assert rel_err(K(g['v']), Kref(g['v'])) < 1e-10


@pytest.mark.gpu
@pytest.mark.parametrize('world', [2, 3])
def test_engine_sharded_preconditioner_virtual_ranks(world):
    """Row-sharded Nystroem factor on the engine (sgdml_b200_assemble_rows, local TRSM / Gram,
    nystroem_project / nystroem_expand), driven for `world` virtual ranks on one GPU: same leverage
    scores and P.v as the reference's unsharded factor."""
    import sgdml_b200
    from sgdml_b200 import dist as sdist
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative, _EngineNystroemOps

    g, task, N, M, R = _setup()
    t = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    d = Desc(N)
    x, gd = d.from_R(R)
    lin = odesc.tril_perms_lin(g['perms'])
    it = Iterative(t, d, float(g['max_memory_gb']), None, False)
    cols, lam, dim_i = g['inducing_pts_idxs'], float(g['lam']), 3 * N
    ops = [_EngineNystroemOps(it, x, gd, lin, task['sig']) for _ in range(world)]
    facs = sdist.run_steps_virtual([sdist.nystroem_factor_steps(ops[r], r, world, M, dim_i, cols, lam) for r in range(world)])
    assert sum(f[0].shape[0] for f in facs) == M * dim_i  # every rank holds only its own rows
    levs = sdist.run_steps_virtual([sdist.lev_scores_steps(ops[r], facs[r][0], len(cols), dim_i) for r in range(world)])
    Pvs = sdist.run_steps_virtual(
        [sdist.precon_apply_steps(ops[r], facs[r][0], len(cols), lam, g['v'], facs[r][1], facs[r][2], dim_i) for r in range(world)]
    )
    for r in range(world):
        assert rel_err(levs[r], g['lev_scores']) < 1e-6
        assert rel_err(Pvs[r], g['Pv']) < 1e-5
        assert np.array_equal(Pvs[r], Pvs[0])


@pytest.mark.gpu
def test_engine_qr_fallback(monkeypatch):
    """iterative.py:312-322 on the engine (shifted CholeskyQR3 on [K_nm; sqrt(lam) I]), forced by making
    the inner Cholesky report failure: same leverage scores and P.v as the reference's factor."""
    import sgdml_b200
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    g, task, N, M, R = _setup()
    t = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    d = Desc(N)
    x, gd = d.from_R(R)
    lin = odesc.tril_perms_lin(g['perms'])
    it = Iterative(t, d, float(g['max_memory_gb']), None, False)
    real = it._cho_factor_stable
    calls = []

    def fake(A, pre_reg=False, eps_mag_max=1):
        if eps_mag_max == -14:
            calls.append(1)
            return False
        return real(A, pre_reg=pre_reg, eps_mag_max=eps_mag_max)

    monkeypatch.setattr(it, '_cho_factor_stable', fake)
    P, lev = it._init_precon_operator(task, x, gd, lin, g['inducing_pts_idxs'])
    assert calls
    assert rel_err(lev, g['lev_scores']) < 1e-6
    assert rel_err(P(g['v']), g['Pv']) < 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize('force_qr', [False, True])
@pytest.mark.parametrize('m', [351, 1107])
def test_engine_nystroem_factor_multi_block(m, force_qr, monkeypatch):
    """The engine's Nystroem factor at m > 128 inducing columns (odd m = 351: three 128-column blocks of TRSM,
    padded square stride m + 1; m = 1107: nine blocks, a Gram matrix spanning two super-tile rows), on a synthetic
    N = 9, M = 150 task: leverage scores and P.v against the oracle's factor on the same columns, through the
    inner Cholesky and through the CholeskyQR3 branch (force_qr).  Both factorisations work on K_mm of
    condition ~1e11, so the two factors agree to conditioning, not to rounding.  Measured on an H100 80GB HBM3
    (400 W), relative to the largest entry: leverage scores 3.1e-9 (m = 351) and 3.3e-8 (m = 1107), P.v 7.0e-9
    and 1.2e-7, the same with and without force_qr; the bounds are ~10x the larger figure."""
    import sgdml_b200
    from sgdml_b200 import synth
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    N, M, sig = 9, 150, 20
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, sig)
    lam = float(task['lam'])
    R = task['R_train'].reshape(M, -1)
    cols = np.sort(np.random.default_rng(m).choice(3 * N * M, m, replace=False))
    v = np.random.default_rng(1).standard_normal(3 * N * M)
    x, gd = odesc.from_R(R)
    lin = odesc.tril_perms_lin(perms)
    B = oiter.nystroem_factor(x, gd, lin, sig, lam, cols, force_qr=force_qr)
    lev_ref, Pv_ref = np.einsum('ij,ij->j', B, B), oiter.precon(B, lam)(v)

    d = Desc(N)
    xe, gde = d.from_R(R)
    it = Iterative(sgdml_b200.GDMLTrain(max_memory=1.0), d, 1.0, None, False)
    if force_qr:
        real, calls = it._cho_factor_stable, []

        def fake(A, pre_reg=False, eps_mag_max=1):
            if eps_mag_max == -14:  # the inner factorisation of iterative.py:305 reports failure
                calls.append(1)
                return False
            return real(A, pre_reg=pre_reg, eps_mag_max=eps_mag_max)

        monkeypatch.setattr(it, '_cho_factor_stable', fake)
    P, lev = it._init_precon_operator(task, xe, gde, lin, cols)
    assert not force_qr or calls
    e_lev, e_pv = rel_err(lev, lev_ref), rel_err(P(v), Pv_ref)
    assert e_lev < 4e-7
    assert e_pv < 1.5e-6


@pytest.mark.gpu
def test_engine_cg_train_matches_reference():
    """GDMLTrain.train with a memory cap that forces the iterative solver, same inducing columns as the
    reference run: converges to the same tolerance in a similar number of iterations and predicts
    the same forces to solver accuracy."""
    import sgdml_b200

    g, task, N, M, R = _setup()
    task['inducing_pts_idxs'] = g['inducing_pts_idxs']
    model = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb'])).train(task)
    assert model['solver_name'] == 'cg'
    assert np.array_equal(model['inducing_pts_idxs'], g['inducing_pts_idxs'])
    assert model['solver_resid'] <= float(g['solver_tol']) * float(g['norm_y_train'])
    assert abs(int(model['solver_iters']) - int(g['solver_iters'])) <= max(5, 0.2 * int(g['solver_iters']))
    E, F = sgdml_b200.GDMLPredict(model).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 2e-3
    assert rel_err(E, g['E_query']) < 2e-3
    # against the analytic solution of the same task the CG model is within solver accuracy too
    exact = sgdml_b200.GDMLTrain().train({k: v for k, v in task.items() if k != 'inducing_pts_idxs'})
    _, F_exact = sgdml_b200.GDMLPredict(exact).predict(g['R_query'])
    assert rel_err(F, F_exact) < 5e-3


@pytest.mark.gpu
def test_engine_cg_own_sampling_converges():
    """Leverage-score sampling path (random inducing columns, iterative.py:353-411)."""
    import sgdml_b200
    from sgdml_b200 import synth

    N, M = 9, 60
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, 20)
    np.random.seed(3)
    model = sgdml_b200.GDMLTrain(max_memory=0.01).train(task)
    assert model['solver_name'] == 'cg' and len(model['inducing_pts_idxs']) % (3 * N) == 0
    exact = sgdml_b200.GDMLTrain().train(task)
    Rq = synth.geometries(N, 20, 1).reshape(20, -1)
    _, F = sgdml_b200.GDMLPredict(model).predict(Rq)
    _, Fx = sgdml_b200.GDMLPredict(exact).predict(Rq)
    assert rel_err(F, Fx) < 5e-3


def _cg_rank(rank, world, port, out_dir):
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
    from sgdml_b200 import synth

    N, M = 9, 60
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, 20)
    np.random.seed(3 + rank)  # different draws per rank: rank 0's inducing columns must win
    trainer = sgdml_b200.GDMLTrain(max_memory=0.01)
    trainer.distributed = True  # every rank trains: sharded Nystroem factor and K.v, agreed solver choice
    model = trainer.train(task)
    # prediction with the sum over training points sharded across the ranks + one all-reduce (SURVEY 8e)
    from conftest import golden_model

    from sgdml_b200 import dist as sdist

    gq = load_golden('n9_m16_s6')
    E_tp, F_tp = sdist.TrainPointShardedPredictor(golden_model(gq), sgdml_b200.GDMLPredict).predict(gq['R_query'])
    F_q = sgdml_b200.GDMLPredict(model).predict(synth.geometries(N, 20, 1).reshape(20, -1))[1]
    np.savez(
        os.path.join(out_dir, 'cg_r%d.npz' % rank),
        alphas=model['alphas_F'],
        idxs=model['inducing_pts_idxs'],
        iters=model['solver_iters'],
        E_tp=E_tp,
        F_tp=F_tp,
        F_q=F_q,
        resid=model['solver_resid'],
        norm_y=model['norm_y_train'],
    )
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_engine_cg_two_ranks_sharded_kv(tmp_path):
    """Two ranks (NCCL): K.v rows sharded + all-gather, Nystroem factor row-sharded (all-reduces of the
    (m x m) matrices and of B v), inducing columns broadcast; both ranks end with the same model, equal
    to the single-rank result with the same columns up to solver accuracy.  Also the prediction
    with training points sharded across the ranks (one all-reduce)."""
    import socket

    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_cg_rank, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0 = np.load(tmp_path / 'cg_r0.npz')
    r1 = np.load(tmp_path / 'cg_r1.npz')
    assert np.array_equal(r0['idxs'], r1['idxs']) and int(r0['iters']) == int(r1['iters'])
    assert rel_err(r1['alphas'], r0['alphas']) < 1e-12
    import sgdml_b200
    from sgdml_b200 import synth

    N, M = 9, 60
    task = synth.make_task(N, M, synth.rotor_swap_group(N, 1, 1), 20)
    task['inducing_pts_idxs'] = r0['idxs']
    single = sgdml_b200.GDMLTrain(max_memory=0.01).train(task)
    # the sharded Gram matrix is summed in a different order, so the two CG runs agree to solver accuracy
    # (tol 1e-4 on the residual), not to rounding
    assert float(r0['resid']) <= 1e-4 * float(r0['norm_y'])
    assert abs(int(single['solver_iters']) - int(r0['iters'])) <= max(5, 0.2 * int(r0['iters']))
    assert rel_err(single['alphas_F'], r0['alphas']) < 2e-2
    F_single = sgdml_b200.GDMLPredict(single).predict(synth.geometries(N, 20, 1).reshape(20, -1))[1]
    assert rel_err(F_single, r0['F_q']) < 2e-3
    gq = load_golden('n9_m16_s6')
    for r in (r0, r1):
        assert rel_err(r['F_tp'], gq['F_query']) < 1e-9
        assert rel_err(r['E_tp'], gq['E_query']) < 1e-9


@pytest.mark.gpu
def test_train_point_sharded_predictor_single_rank():
    import sgdml_b200
    from conftest import golden_model
    from sgdml_b200 import dist as sdist

    gq = load_golden('n9_m16_s6')
    model = golden_model(gq)
    E, F = sdist.TrainPointShardedPredictor(model, sgdml_b200.GDMLPredict).predict(gq['R_query'])
    assert rel_err(F, gq['F_query']) < 1e-9 and rel_err(E, gq['E_query']) < 1e-9
    M = model['R_desc'].shape[1]
    parts = [sgdml_b200.GDMLPredict(sdist.model_shard(model, lo, hi)).predict(gq['R_query']) for lo, hi in [(0, 7), (7, M)]]
    F_sum = (parts[0][1] + parts[1][1]) * float(model['std'])
    assert rel_err(F_sum, gq['F_query']) < 1e-9


# --------------------------------------------------------------------------- device-resident PCG through the C ABI
def _pcg_call(pred, X, m, lam, y, x0, tol_abs, max_iters, check_every=5, exchange=None, progress=None):
    import ctypes

    import torch

    from sgdml_b200 import _lib

    L = _lib.lib()
    n = y.size
    n_train = pred.n_train
    n_rows = n
    wsd = int(L.sgdml_b200_pcg_workspace_doubles(n, n_rows, m, check_every))
    ws = torch.empty(wsd, dtype=torch.float64, device='cuda')
    x = np.zeros(n) if x0 is None else np.array(x0, dtype=np.float64)
    iters, resid = ctypes.c_int64(0), ctypes.c_double(0.0)
    exch = _lib.EXCHANGE_FN(exchange) if exchange is not None else ctypes.cast(None, _lib.EXCHANGE_FN)
    prog = _lib.PROGRESS_FN(progress) if progress is not None else ctypes.cast(None, _lib.PROGRESS_FN)
    _lib.check(
        L.sgdml_b200_pcg(
            pred._handle, 0, n_train, X.data_ptr() if m else None, m, X.shape[1] if m else 0, float(lam), _lib.ptr(y), _lib.ptr(x),
            1 if x0 is None else 0, float(tol_abs), int(max_iters), int(check_every), ws.data_ptr(), wsd, exch, None, prog, None,
            ctypes.byref(iters), ctypes.byref(resid), _lib.current_stream(),
        ),
        'pcg',
    )
    return x, int(iters.value), float(resid.value)


def _np_pcg(A, Pinv, y, x0, n_iters):
    """Textbook PCG (the loop of scipy.sparse.linalg.cg the reference calls, iterative.py:740-752)."""
    x = np.zeros_like(y) if x0 is None else x0.copy()
    r = y - A @ x
    z = Pinv(r)
    p = z.copy()
    rz = r @ z
    hist = []
    for _ in range(n_iters):
        Ap = A @ p
        alpha = rz / (p @ Ap)
        x += alpha * p
        r -= alpha * Ap
        hist.append(np.linalg.norm(r))
        z = Pinv(r)
        rz_new = r @ z
        p = z + (rz_new / rz) * p
        rz = rz_new
    return x, np.array(hist)


@pytest.mark.gpu
@pytest.mark.parametrize('precon', [False, True])
@pytest.mark.parametrize('warm', [False, True])
def test_pcg_c_abi_matches_numpy_cg(precon, warm):
    """sgdml_b200_pcg against a NumPy PCG on the EXPLICIT system matrix of a reference fixture: same iterates."""
    import sgdml_b200
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    g, task, N, M, R = _setup()
    lam = float(g['lam'])
    d = Desc(N)
    x_desc, gd = d.from_R(R)
    lin = odesc.tril_perms_lin(g['perms'])
    t = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    it = Iterative(t, d, float(g['max_memory_gb']), None, False)
    n = 3 * N * M
    it._init_kernel_operator(task, x_desc, gd, lin, lam, n)
    from oracle import assemble as oassemble

    K = oassemble.assemble(x_desc, gd, lin, int(g['sig']))
    A = -K + lam * np.eye(n)
    y = np.ascontiguousarray(g['y'], dtype=np.float64)
    if precon:
        P, _ = it._init_precon_operator(task, x_desc, gd, lin, g['inducing_pts_idxs'])
        X, m = P.factor[0], P.factor[1]
        Xh = X[:, :m].cpu().numpy()
        Pinv = lambda v: (Xh @ (Xh.T @ v) - v) / lam  # noqa: E731  (iterative.py:136-138)
    else:
        X, m = None, 0
        Pinv = lambda v: v.copy()  # noqa: E731
    x0 = 0.01 * np.random.default_rng(5).standard_normal(n) if warm else None
    n_it = 12
    x_ref, hist_ref = _np_pcg(A, Pinv, y, x0, n_it)
    seen = []

    def progress(_ctx, iters_done, hist, n_new):
        seen.extend(hist[i] for i in range(n_new))
        return 0

    x, iters, resid = _pcg_call(it.gdml_predict, X, m, lam, y, x0, 0.0, n_it, check_every=5, progress=progress)
    assert iters == n_it and len(seen) == n_it
    # CG on a system of condition ~1e11 amplifies rounding differences from iteration to iteration (measured: 3e-5
    # after 12 unpreconditioned iterations): the first iterations must agree to rounding, the rest to 1e-3
    assert rel_err(np.array(seen[:5]), hist_ref[:5]) < 1e-6
    assert rel_err(np.array(seen), hist_ref) < 1e-3
    assert rel_err(x, x_ref) < 1e-2
    assert abs(resid - hist_ref[-1]) < 1e-3 * hist_ref[-1]


@pytest.mark.gpu
def test_pcg_stops_at_tolerance_and_on_request():
    """The device-side freeze: x stops changing at the first iteration below the tolerance, even inside a chunk;
    a non-zero return of the progress function ends the solve; the exchange hook is called in stream order."""
    import sgdml_b200
    from sgdml_b200.desc import Desc
    from sgdml_b200.solvers.iterative import Iterative

    g, task, N, M, R = _setup()
    lam = float(g['lam'])
    d = Desc(N)
    x_desc, gd = d.from_R(R)
    lin = odesc.tril_perms_lin(g['perms'])
    t = sgdml_b200.GDMLTrain(max_memory=float(g['max_memory_gb']))
    it = Iterative(t, d, float(g['max_memory_gb']), None, False)
    n = 3 * N * M
    it._init_kernel_operator(task, x_desc, gd, lin, lam, n)
    P, _ = it._init_precon_operator(task, x_desc, gd, lin, g['inducing_pts_idxs'])
    X, m = P.factor[0], P.factor[1]
    y = np.ascontiguousarray(g['y'], dtype=np.float64)
    tol_abs = 1e-4 * np.linalg.norm(y)
    hist = []

    def progress(_ctx, iters_done, h, n_new):
        hist.extend(h[i] for i in range(n_new))
        return 0

    calls = []

    def exchange(_ctx, op, buf, count):  # single rank: nothing to exchange, but every call is recorded
        calls.append((op, count))
        return 0

    x, iters, resid = _pcg_call(it.gdml_predict, X, m, lam, y, None, tol_abs, 10000, check_every=50, exchange=exchange, progress=progress)
    assert resid <= tol_abs and iters == len(hist)
    assert all(h > tol_abs for h in hist[:-1]) and hist[-1] <= tol_abs  # stopped AT the first converged iteration
    assert abs(iters - int(g['solver_iters'])) <= max(5, 0.2 * int(g['solver_iters']))
    assert (0, m) in calls and (1, n) in calls and len(calls) >= 3 * iters
    # the frozen x reproduces the reported residual
    K = it._init_kernel_operator(task, x_desc, gd, lin, lam, n)
    r = y + K(x)  # A x = -K_op(x)
    assert abs(np.linalg.norm(r) - resid) < 1e-6 * resid + 1e-9

    def stop_after_three(_ctx, iters_done, h, n_new):
        return 1 if iters_done >= 3 else 0

    _, iters2, _ = _pcg_call(it.gdml_predict, X, m, lam, y, None, 0.0, 1000, check_every=1, progress=stop_after_three)
    assert iters2 == 3
