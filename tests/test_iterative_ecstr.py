"""Nystroem-preconditioned CG with energy constraints in the kernel (use_E_cstr), CPU side: the oracle against the
reference's own energy-constrained iterative solve frozen in tests/golden/cg_ecstr_n9_m40.npz, and the row-sharded
factor / leverage scores / P.v of sgdml_b200.dist in the (3NM + M) layout [forces; energies]."""

import os
import sys

import numpy as np
import pytest

import ecstr_oracle as eoracle
from conftest import ROOT, load_golden, rel_err
from test_dist_gloo import NumpyNystroemOps, _free_port

from oracle import assemble as oassemble
from oracle import desc as odesc
from oracle import iterative as oiter
from oracle import predict as opredict


def iters_close(iters, ref_iters, frac=0.2):
    """The iteration-count bound of test_iterative: within max(5, frac * ref_iters) of the reference's run."""
    return abs(iters - ref_iters) <= max(5, frac * ref_iters)


def setup_ecstr():
    """(g, task, N, M, R_desc, R_d_desc, tril_perms_lin) of the fixture; the task has use_E_cstr set."""
    from sgdml_b200 import synth

    g = load_golden('cg_ecstr_n9_m40')
    N, M = int(g['n_atoms']), int(g['n_train'])
    task = synth.make_task(N, M, g['perms'], int(g['sig']), lam=float(g['lam']))
    task['use_E_cstr'] = True
    x, gd = odesc.from_R(task['R_train'].reshape(M, -1))
    return g, task, N, M, x, gd, odesc.tril_perms_lin(g['perms'])


def model_like_ecstr(g, task, R_desc, R_d_desc, alphas):
    """Model dict of the energy-constrained coefficients alphas = [alphas_F; alphas_E]."""
    N, M = int(g['n_atoms']), R_desc.shape[0]
    a_F, a_E = alphas[:-M], alphas[-M:]
    return {
        'type': 'm',
        'z': task['z'],
        'R_desc': R_desc.T,
        'R_d_desc_alpha': odesc.d_desc_dot_vec(R_d_desc, a_F.reshape(-1, 3 * N)),
        'alphas_F': a_F,
        'alphas_E': a_E,
        'c': float(g['c']),
        'std': float(g['std']),
        'sig': int(g['sig']),
        'lam': float(g['lam']),
        'perms': g['perms'],
        'tril_perms_lin': odesc.tril_perms_lin(g['perms']),
        'use_E': True,
    }


def test_fixture_has_energy_columns():
    g = load_golden('cg_ecstr_n9_m40')
    n_f = 3 * int(g['n_atoms']) * int(g['n_train'])
    assert np.any(g['inducing_pts_idxs'] >= n_f)
    assert g['K_nm'].shape == (n_f + int(g['n_train']), len(g['inducing_pts_idxs']))


def test_oracle_ecstr_columns_match_reference():
    g, task, N, M, x, gd, lin = setup_ecstr()
    K = oassemble.assemble_E_cstr(x, gd, lin, int(g['sig']))
    assert rel_err(K[:, g['inducing_pts_idxs']], g['K_nm']) < 1e-12


def test_oracle_ecstr_preconditioner_and_solve():
    g, task, N, M, x, gd, lin = setup_ecstr()
    lam, sig = float(g['lam']), int(g['sig'])
    B = eoracle.nystroem_factor_ecstr(x, gd, lin, sig, lam, g['inducing_pts_idxs'])
    assert B.shape[1] == 3 * N * M + M
    assert rel_err(np.einsum('ij,ij->j', B, B), g['lev_scores']) < 1e-6
    assert rel_err(oiter.precon(B, lam)(g['v']), g['Pv']) < 1e-5
    zeros = np.zeros(3 * N * M + M)
    alphas, info, iters, _ = eoracle.solve_ecstr(model_like_ecstr(g, task, x, gd, zeros), x, gd, lin, sig, lam, g['y'], g['inducing_pts_idxs'])
    assert info == 0
    # CG on this system (condition ~1e11) is sensitive to rounding: the reference's run takes 146 iterations,
    # scipy.sparse.linalg.cg on the oracle's operators (leverage scores, P.v and K.v match the reference's) 115, 21 %
    # fewer -- hence 25 % here, and the 20 % of test_iterative for the engine (measured on an H100: 166)
    assert iters_close(iters, int(g['solver_iters_fixed_cols']), frac=0.25)
    E, F = opredict.Predictor(model_like_ecstr(g, task, x, gd, alphas)).predict(g['R_query'])
    assert rel_err(F, g['F_query']) < 2e-3  # both are converged to rtol 1e-4 only
    assert rel_err(E, g['E_query']) < 2e-3


def test_oracle_ecstr_kernel_op_is_the_matrix():
    """kernel_op_ecstr (predictor with alphas_E, [F; -E] - lam v) is the explicit (3NM + M) matrix."""
    g, task, N, M, x, gd, lin = setup_ecstr()
    lam = float(g['lam'])
    K = oassemble.assemble_E_cstr(x, gd, lin, int(g['sig']))
    Kop = eoracle.kernel_op_ecstr(model_like_ecstr(g, task, x, gd, np.zeros(3 * N * M + M)), x, gd, lam)
    assert rel_err(Kop(g['v']), K @ g['v'] - lam * g['v']) < 1e-10


class NumpyNystroemOpsEcstr(NumpyNystroemOps):
    """NumpyNystroemOps on the energy-constrained matrix: a rank's block is the force rows of its training points,
    then their energy rows (sgdml_b200_assemble_ecstr_rows)."""

    def __init__(self, g, K_full, dim_i):
        super().__init__(g)
        self.K_full, self.dim_i = K_full, dim_i

    def assemble_rows(self, lo, hi, cols):
        import torch

        n_f = self.K_full.shape[0] // (self.dim_i + 1) * self.dim_i
        rows = np.concatenate([np.arange(lo * self.dim_i, hi * self.dim_i), n_f + np.arange(lo, hi)])
        return torch.from_numpy(np.ascontiguousarray(self.K_full[rows][:, cols]))


def sharded_cols(g):
    """The fixture's inducing columns plus the energy column of point 35, which a non-zero rank owns for world 2
    and 3 (the fixture's own energy columns, points 16 and 17, are rank 0's for world 2)."""
    n_f = 3 * int(g['n_atoms']) * int(g['n_train'])
    return np.union1d(g['inducing_pts_idxs'], [n_f + 35])


@pytest.mark.parametrize('force_qr', [False, True])
def test_virtual_ranks_ecstr_match_unsharded(force_qr):
    """dist.nystroem_factor_steps / lev_scores_steps / precon_apply_steps with use_E_cstr on 1, 2 and 3 virtual
    ranks (M = 40: uneven shards for 3) against the unsharded oracle factor; the QR fallback's shift uses the full
    row count 3NM + M."""
    from sgdml_b200 import dist as sdist

    g, task, N, M, x, gd, lin = setup_ecstr()
    lam, dim_i = float(g['lam']), 3 * N
    cols = sharded_cols(g)
    B = eoracle.nystroem_factor_ecstr(x, gd, lin, int(g['sig']), lam, cols, force_qr=force_qr)
    lev_ref, Pv_ref = np.einsum('ij,ij->j', B, B), oiter.precon(B, lam)(g['v'])
    K_full = oassemble.assemble_E_cstr(x, gd, lin, int(g['sig']))
    for world in (1, 2, 3):
        ops = [NumpyNystroemOpsEcstr(g, K_full, dim_i) for _ in range(world)]
        for o in ops:
            o.force_qr = force_qr
        facs = sdist.run_steps_virtual(
            [sdist.nystroem_factor_steps(ops[r], r, world, M, dim_i, cols, lam, use_E_cstr=True) for r in range(world)]
        )
        assert sum(f[0].shape[0] for f in facs) == M * (dim_i + 1)
        lo, hi = sdist.shard_bounds(M, world, world - 1)
        assert world == 1 or lo <= 35 < hi  # the extra energy column lives on the last rank
        # the sharded factor is the unsharded one's rows, split by rank (the QR branch's R factor is defined up to the
        # signs of its rows, so there only B^T B-invariant quantities are compared)
        for r in range(world if not force_qr else 0):
            lo, hi = facs[r][1], facs[r][2]
            rows = np.concatenate([np.arange(lo * dim_i, hi * dim_i), dim_i * M + np.arange(lo, hi)])
            assert rel_err(facs[r][0].numpy()[:, : len(cols)], B.T[rows]) < 1e-6
        levs = sdist.run_steps_virtual(
            [sdist.lev_scores_steps(ops[r], facs[r][0], len(cols), dim_i, use_E_cstr=True) for r in range(world)]
        )
        Pvs = sdist.run_steps_virtual(
            [
                sdist.precon_apply_steps(ops[r], facs[r][0], len(cols), lam, g['v'], facs[r][1], facs[r][2], dim_i, use_E_cstr=True)
                for r in range(world)
            ]
        )
        for r in range(world):
            assert rel_err(levs[r], lev_ref) < 1e-6
            assert rel_err(Pvs[r], Pv_ref) < 1e-6


def _exchange_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist

    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from sgdml_b200 import dist as sdist

    out = {}
    for n_pts in (8, 7):  # equal and ragged shards
        di = 3
        n_f = n_pts * di
        ws = torch.zeros(2 + n_f + n_pts + 3, dtype=torch.float64)
        lo, hi = sdist.shard_bounds(n_pts, world, rank)
        full_f = np.arange(n_f, dtype=np.float64) + 100.0
        full_e = -np.arange(n_pts, dtype=np.float64) - 1.0
        ws[2 + lo * di : 2 + hi * di] = torch.from_numpy(full_f[lo * di : hi * di])  # only the owned rows are valid
        ws[2 + n_f + lo : 2 + n_f + hi] = torch.from_numpy(full_e[lo:hi])
        sdist.exchange_on_workspace(ws, 2, n_f, 1, n_pts, di)  # force part
        sdist.exchange_on_workspace(ws, 2 + n_f, n_pts, 2, n_pts, di)  # energy tail
        out['ws%d' % n_pts] = ws.numpy().copy()
    np.savez(os.path.join(out_dir, 'x%d.npz' % rank), **out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(180)
def test_exchange_op2_two_rank_gloo(tmp_path):
    """The exchange of sgdml_b200_pcg_ecstr on torch.distributed: op 1 on the force part, op 2 on the M-entry
    energy tail, with equal (8 points) and uneven (7 points) shards; nothing outside the two buffers changes."""
    import torch.multiprocessing as mp

    mp.spawn(_exchange_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        with np.load(tmp_path / ('x%d.npz' % r)) as f:
            for n_pts in (8, 7):
                ws = f['ws%d' % n_pts]
                n_f = 3 * n_pts
                assert not ws[:2].any() and not ws[2 + n_f + n_pts :].any()
                assert np.array_equal(ws[2 : 2 + n_f], np.arange(n_f) + 100.0)
                assert np.array_equal(ws[2 + n_f : 2 + n_f + n_pts], -np.arange(n_pts) - 1.0)

