"""CPU, world_size 2, gloo: virials from the sharded predictors -- TrainPointShardedPredictor.predict_virial (the sum
over training points split, one all-reduce of [F | E | W]) and dist.predict_virial_sharded (queries and their
per-geometry cells split) -- with the oracle as the injected predictor, checked against the oracle virial of the
unsharded model in each geometry's cell.  Also: model_shard slices alphas_E, so the shards of an energy-constrained
model add up."""

import os
import sys

import numpy as np
import pytest

import predict_checks as pc
import virial_cells_checks as vcc
import virial_checks as vc
from conftest import ROOT
from test_dist_gloo import _free_port

N, M, B = 9, 13, 7


def _models():
    lat = pc.skewed_cell(N)
    return {
        'free': vc.make_model(N, M, seed=11),
        'pbc': vc.make_model(N, M, seed=12, lattice=lat),
        'ecstr': vc.make_model(N, M, seed=13, ecstr=True, lattice=lat),
    }


def _queries():
    R = vc.queries(N, B, 21)
    cells = vcc.cells_for(R, pc.skewed_cell(N), 22)
    return R, cells


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import torch.distributed as dist

    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from sgdml_b200 import dist as sdist

    R, cells = _queries()
    res = {}
    for name, model in _models().items():
        tp = sdist.TrainPointShardedPredictor(model, vcc.OracleVirialPredictor)
        assert (tp.hi - tp.lo) < M  # every rank holds a proper part of the training points
        res[name + '_own'] = tp.predict_virial(R)  # the model's own cell (none for the free model)
        res[name + '_cells'] = tp.predict_virial(R, lattice=cells)
    F_only = tp.predict_virial(R, lattice=cells, return_E=False)
    assert len(F_only) == 2 and np.array_equal(F_only[1], res['ecstr_cells'][2])
    full = vcc.OracleVirialPredictor(_models()['pbc'])
    res['sharded_cells'] = sdist.predict_virial_sharded(lambda r, lat: full.predict_virial(r, lattice=lat), R, cells)
    lo, hi, E_l, F_l, W_l = sdist.predict_virial_sharded(
        lambda r, lat: full.predict_virial(r, lattice=lat), R, cells, gather=False)
    assert (lo, hi) == sdist.shard_bounds(B, world, rank) and W_l.shape == (hi - lo, 3, 3)
    np.savez(os.path.join(out_dir, 'r%d.npz' % rank),
             **{'%s_%s' % (k, c): v for k, t in res.items() for c, v in zip('EFW', t)})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_gloo_virial(tmp_path):
    import torch.multiprocessing as mp

    from oracle import predict as opredict

    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    R, cells = _queries()
    vcc.assert_cells_wrap_differently(R, cells)
    models = _models()
    for r in range(2):
        with np.load(tmp_path / ('r%d.npz' % r)) as f:
            for name, model in models.items():
                op = opredict.Predictor(model)
                for case, cc in (('own', None), ('cells', cells)):
                    k = '%s_%s' % (name, case)
                    vcc.check_cells('rank %d train-point sharded %s' % (r, k), model, op, R, cc,
                                    f[k + '_E'], f[k + '_F'], f[k + '_W'])
            vcc.check_cells('rank %d query sharded, cells' % r, models['pbc'], opredict.Predictor(models['pbc']), R,
                            cells, f['sharded_cells_E'], f['sharded_cells_F'], f['sharded_cells_W'])
    with np.load(tmp_path / 'r0.npz') as f0, np.load(tmp_path / 'r1.npz') as f1:
        for k in f0.files:
            assert np.array_equal(f0[k], f1[k]), '%s differs between the ranks' % k


def test_model_shards_add_up_energy_constrained():
    """Shards of an energy-constrained model (alphas_E sliced with the training points) sum to the unsharded E and F."""
    from oracle import predict as opredict
    from sgdml_b200 import dist as sdist

    model = _models()['ecstr']
    R = vc.queries(N, 5, 31, model['lattice'])
    E_ref, F_ref = opredict.Predictor(model).predict(R)
    E = np.zeros(R.shape[0])
    F = np.zeros_like(F_ref)
    for lo, hi in [(0, 5), (5, 6), (6, M)]:
        sub = sdist.model_shard(model, lo, hi)
        assert np.array_equal(sub['alphas_E'], model['alphas_E'][lo:hi])
        e, f = opredict.Predictor(sub).predict(R)
        E += e
        F += f
    std, c = float(model['std']), float(model['c'])
    assert np.max(np.abs(F * std - F_ref)) < 1e-10 * np.max(np.abs(F_ref))
    assert np.max(np.abs(E * std + c - E_ref)) < 1e-10 * np.max(np.abs(E_ref))


def test_stacked_inverses_match_single_cell_inverses():
    """GDMLPredict.predict_virial inverts a (B, 3, 3) stack of cells in one np.linalg.inv call; each inverse is
    bit-identical to the one the single-cell call computes, so all-equal cells give the single-cell results bit for
    bit."""
    import torch

    from sgdml_b200.predict import cells_and_inverses

    rng = np.random.default_rng(5)
    base = pc.skewed_cell(21) * 1.6
    cells = np.stack([(np.eye(3) + 0.1 * rng.standard_normal((3, 3))) @ base for _ in range(257)])
    lat, inv = cells_and_inverses(cells)
    assert lat.flags['C_CONTIGUOUS'] and inv.flags['C_CONTIGUOUS'] and inv.shape == (257, 3, 3)
    for b in range(cells.shape[0]):
        l1, i1 = cells_and_inverses(cells[b])
        assert np.array_equal(l1, lat[b]) and np.array_equal(i1, inv[b]), 'cell %d' % b
    lt, it = cells_and_inverses(torch.from_numpy(cells))
    assert np.array_equal(lt, lat) and np.array_equal(it, inv)
    for bad in (np.eye(2), np.zeros((4, 3, 2)), np.zeros((2, 2, 3, 3))):
        with pytest.raises(ValueError):
            cells_and_inverses(bad)
