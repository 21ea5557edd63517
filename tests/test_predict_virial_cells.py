"""sgdml_b200_predict_virial_cells / GDMLPredict.predict_virial with a (B, 3, 3) lattice: one cell per geometry on every
batch route of tests/test_predict_virial.py, against the oracle evaluated in each geometry's own cell (check_predict /
check_W at a 10x margin).  Every geometry gets its own random skewed cell, and pairs wrap into different images in
different geometries.  All-equal cells give the single-cell call's E, F and W bit for bit on every route; new cells
replay the graph (the main-kernel launch counter does not move); rejected calls change nothing.  Also the training-point
virial (predict_virial(R=None)) and TrainPointShardedPredictor.predict_virial on one GPU."""

import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import predict_checks as pc  # noqa: E402
import virial_cells_checks as vcc  # noqa: E402
import virial_checks as vc  # noqa: E402
from conftest import load_golden  # noqa: E402
from oracle import desc as odesc  # noqa: E402
from oracle import predict as opredict  # noqa: E402
from test_predict_bulk import _chunk_cap, _main_launches  # noqa: E402

ERR_ARG = -1000
SHAPES = {'d36': (9, 70), 'd105': (15, 41), 'd253': (23, 29), 'd276': (24, 19)}


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


@contextlib.contextmanager
def _env(monkeypatch, **kv):
    with monkeypatch.context() as mp:
        for k, v in kv.items():
            mp.setenv(k, v)
        yield


def _np(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def _nan(B, dim_i):
    return np.full(B, np.nan), np.full((B, dim_i), np.nan), np.full((B, 3, 3), np.nan)


def _same(a, b):
    return all(np.array_equal(_np(x), _np(y)) for x, y in zip(a, b))


def _routes(eng, monkeypatch, model, op, base, Rq, tag, seed, pipelined_B=4100):
    """Every batch route with one cell per geometry; on each, all-equal cells (= base) against the single-cell call."""
    import torch

    N = int(np.asarray(model['z']).shape[0])
    dim_i = 3 * N
    stack = lambda B: np.repeat(base[None], B, axis=0)  # noqa: E731
    p = eng.GDMLPredict(model)
    # host B = 37 (plain launches), out= NaN-filled
    R = Rq(37, 0)
    cells = vcc.cells_for(R, base, seed)
    vcc.assert_cells_wrap_differently(R, cells)
    out = _nan(37, dim_i)
    E, F, W = p.predict_virial(R, lattice=cells, out=out)
    assert E is out[0] and W is out[2]
    vcc.check_cells('%s host B=37' % tag, model, op, R, cells, E, F, W)
    assert _same(p.predict_virial(R, lattice=stack(37)), p.predict_virial(R, lattice=base)), tag
    # CUDA tensors B = 1 and 37 (host cells, a torch stack too), pinned host tensors B = 20
    for B, s in ((1, 1), (37, 2)):
        R = Rq(B, s)
        cells = vcc.cells_for(R, base, seed + s)
        Rt = torch.from_numpy(R).cuda()
        E, F, W = p.predict_virial(Rt, lattice=torch.from_numpy(cells))
        torch.cuda.synchronize()
        assert W.is_cuda and W.shape == (B, 3, 3)
        vcc.check_cells('%s device B=%d' % (tag, B), model, op, R, cells, _np(E), _np(F), _np(W))
        a, b = p.predict_virial(Rt, lattice=stack(B)), p.predict_virial(Rt, lattice=base)
        torch.cuda.synchronize()
        assert _same(a, b), '%s device B=%d: equal cells differ from the single-cell call' % (tag, B)
    R = Rq(20, 3)
    cells = vcc.cells_for(R, base, seed + 3)
    E, F, W = p.predict_virial(torch.from_numpy(R).pin_memory(), lattice=cells)
    assert W.is_pinned() and F.is_pinned()
    vcc.check_cells('%s pinned B=20' % tag, model, op, R, cells, _np(E), _np(F), _np(W))
    # several chunks of at most 5 queries
    with _chunk_cap(5):
        pc5 = eng.GDMLPredict(model)
        R = Rq(23, 4)
        cells = vcc.cells_for(R, base, seed + 4)
        E, F, W = pc5.predict_virial(R, lattice=cells)
        assert _same(pc5.predict_virial(R, lattice=stack(23)), pc5.predict_virial(R, lattice=base))
    vcc.check_cells('%s host B=23 cap 5' % tag, model, op, R, cells, E, F, W)
    # B = 1, 3, 16: plain launches and both graph forms, bit-identical; new cells replay the graph
    for B in (1, 3, 16):
        R = Rq(B, 10 + B)
        cells = vcc.cells_for(R, base, seed + 10 + B)
        with _env(monkeypatch, SGDML_B200_GRAPH='0'):
            E0, F0, W0 = eng.GDMLPredict(model).predict_virial(R, lattice=cells)
        vcc.check_cells('%s host B=%d plain' % (tag, B), model, op, R, cells, E0, F0, W0)
        for zc in ('1', '0'):
            with _env(monkeypatch, SGDML_B200_GRAPH='1', SGDML_B200_GRAPH_ZEROCOPY=zc):
                pg = eng.GDMLPredict(model)
                R1 = Rq(B, 20 + B)
                pg.predict_virial(R1, lattice=vcc.cells_for(R1, base, seed + 20 + B))  # captures
                n0 = _main_launches()
                E, F, W = pg.predict_virial(R, lattice=cells, out=_nan(B, dim_i))  # replays with new cells
                assert _main_launches() == n0, 'graph not replayed'
                # all-equal cells against the single-cell call, both replaying the same graph
                for _ in range(2):
                    a, b = pg.predict_virial(R, lattice=stack(B)), pg.predict_virial(R, lattice=base)
                assert _same(a, b), '%s B=%d zero copy %s: equal cells differ from the single-cell call' % (tag, B, zc)
            assert np.array_equal(E, E0) and np.array_equal(F, F0) and np.array_equal(W, W0), \
                '%s B=%d: graph (zero copy %s) differs from plain launches' % (tag, B, zc)
    # pipelined host batch: chunk edges and sampled rows against the oracle
    if pipelined_B:
        B = pipelined_B
        R = Rq(B, 40)
        rows = np.unique(np.concatenate([[0, 1024, 1025, 2049, 3075, B - 1],
                                         np.random.default_rng(seed).choice(B, 24, replace=False)]))
        cells = vcc.cells_for(R, base, seed + 40, rows=rows)
        E, F, W = p.predict_virial(R, lattice=cells)
        vcc.check_cells('%s pipelined B=%d (%d rows)' % (tag, B, len(rows)), model, op, R[rows], cells[rows],
                        E[rows], F[rows], W[rows])
        assert _same(p.predict_virial(R, lattice=stack(B)), p.predict_virial(R, lattice=base)), tag
    return p


def _periodic(name, seed, ecstr=False):
    N, M = SHAPES[name]
    base = pc.skewed_cell(N)
    model = vc.make_model(N, M, seed=seed, lattice=base, ecstr=ecstr)
    return N, base, model


N_SEED = {'d36': 101, 'd105': 102, 'd253': 103, 'd276': 104}


@pytest.mark.parametrize('name', sorted(SHAPES))
def test_cells_every_route(eng, monkeypatch, name):
    N, base, model = _periodic(name, N_SEED[name])
    op = opredict.Predictor(model)
    _routes(eng, monkeypatch, model, op, base, lambda B, s: vc.queries(N, B, 700 + s), 'cells %s' % name, 700)


def test_cells_energy_constrained(eng, monkeypatch):
    N, base, model = _periodic('d105', 111, ecstr=True)
    op = opredict.Predictor(model)
    _routes(eng, monkeypatch, model, op, base, lambda B, s: vc.queries(N, B, 800 + s), 'cells ecstr d105', 800)


def test_cells_long_descriptors_n240(eng, monkeypatch):
    """N = 240, M = 2 (D = 28 680): the k_fdesc_gather<true> / k_fdesc_project<true> finishing pair with per-geometry cells."""
    g = load_golden('big_n240_m2_s3')
    N = int(g['n_atoms'])
    M = g['R_train'].shape[0]
    x, gd = odesc.from_R(g['R_train'].reshape(M, -1))
    model = {
        'type': 'm', 'z': g['z'], 'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(gd, g['alphas_F'].reshape(M, -1)), 'alphas_F': g['alphas_F'],
        'c': float(g['c']), 'std': float(g['std']), 'sig': int(g['sig']), 'lam': float(g['lam']), 'perms': g['perms'],
        'tril_perms_lin': odesc.tril_perms_lin(g['perms']), 'use_E': True,
    }
    Rg = np.ascontiguousarray(g['R_query']).reshape(-1, 3 * N)
    r = Rg.reshape(Rg.shape[0], N, 3)
    ext = np.max(r.max(axis=1) - r.min(axis=1), axis=0)  # the geometries' extent per axis
    base = np.array([[1.0, 0.12, -0.08], [0.0, 0.99, 0.1], [0.0, 0.0, 0.99]]) * (0.8 * np.max(ext))
    rng = np.random.default_rng(9)

    def Rq(B, s):  # the fixture's queries, jiggled
        idx = np.random.default_rng(s).integers(0, Rg.shape[0], B)
        return np.ascontiguousarray(Rg[idx] + 0.02 * rng.standard_normal((B, 3 * N)))

    op = opredict.Predictor(model)
    _routes(eng, monkeypatch, model, op, base, Rq, 'cells n240', 900, pipelined_B=0)


def test_cells_pipelined_energy_constrained_d276(eng):
    """The pipelined host path (B = 4100, four chunks on two streams) on the GEMM-composed shape with alphas_E: chunk
    edges and sampled rows against the oracle."""
    N, base, model = _periodic('d276', 121, ecstr=True)
    op = opredict.Predictor(model)
    p = eng.GDMLPredict(model)
    B = 4100
    R = vc.queries(N, B, 122)
    rows = np.unique(np.concatenate([[0, 1024, 1025, 2049, 3075, B - 1],
                                     np.random.default_rng(4).choice(B, 24, replace=False)]))
    cells = vcc.cells_for(R, base, 123, rows=rows)
    E, F, W = p.predict_virial(R, lattice=cells)
    vcc.check_cells('pipelined ecstr d276', model, op, R[rows], cells[rows], E[rows], F[rows], W[rows])


def test_rejected_cells_change_nothing(eng):
    """One singular cell among B, one NaN cell, B - 1 cells, device cell pointers: rejected before any work; the NaN
    outputs, the model's cell, its captured graph and later results stay bit for bit as they were."""
    import torch

    from sgdml_b200 import _lib

    N, base, model = _periodic('d36', 131)
    p = eng.GDMLPredict(model)
    B = 3
    R = vc.queries(N, B, 132)
    cells = vcc.cells_for(R, base, 133)
    inv = np.ascontiguousarray(np.linalg.inv(cells))
    E0, F0, W0 = p.predict_virial(R, lattice=cells)  # captures
    Em, Fm = p.predict(R)
    n0 = _main_launches()
    L = _lib.lib()
    st = _lib.current_stream()
    sing = cells.copy()
    sing[1] = np.outer([1.0, 2.0, 3.0], [1.0, 0.5, 0.25])
    nanc = cells.copy()
    nanc[2, 1, 1] = np.nan
    cd, idv = torch.from_numpy(cells).cuda(), torch.from_numpy(inv).cuda()
    out = _nan(B, 3 * N)
    for a, b in ((_lib.ptr(sing), _lib.ptr(inv)), (_lib.ptr(nanc), _lib.ptr(inv)), (cd.data_ptr(), idv.data_ptr()),
                 (_lib.ptr(cells), idv.data_ptr()), (_lib.ptr(cells), None)):
        rc = L.sgdml_b200_predict_virial_cells(p._handle, _lib.ptr(R), B, a, b, _lib.ptr(out[0]), _lib.ptr(out[1]),
                                               _lib.ptr(out[2]), st)
        assert rc == ERR_ARG
    with pytest.raises(np.linalg.LinAlgError):  # np.linalg.inv of the stack, as for a singular single cell
        p.predict_virial(R, lattice=sing, out=out)
    with pytest.raises(_lib.EngineError):
        p.predict_virial(R, lattice=nanc, out=out)
    with pytest.raises(ValueError):
        p.predict_virial(R, lattice=cells[: B - 1], out=out)
    assert all(np.all(np.isnan(o)) for o in out), 'a rejected call wrote output'
    E1, F1, W1 = p.predict_virial(R, lattice=cells)
    assert _main_launches() == n0, 'a rejected call dropped the captured graph'
    assert np.array_equal(E1, E0) and np.array_equal(F1, F0) and np.array_equal(W1, W0)
    E2, F2 = p.predict(R)
    assert np.array_equal(E2, Em) and np.array_equal(F2, Fm), 'a rejected call changed the model'


@pytest.mark.parametrize('kind', ['free', 'pbc', 'ecstr'])
def test_train_point_virial(eng, kind):
    """predict_virial(R=None): the training points from the cached descriptors, against the oracle virial of R_train in
    the model's cell; E and F bit-identical to predict(R=None); a lattice is refused."""
    from sgdml_b200 import synth

    N, M = SHAPES['d36']
    base = pc.skewed_cell(N) if kind != 'free' else None
    seed = {'free': 141, 'pbc': 142, 'ecstr': 143}[kind]
    model = vc.make_model(N, M, seed=seed, lattice=base, ecstr=kind == 'ecstr')
    R_train = synth.geometries(N, M, seed).reshape(M, -1)
    if base is not None:
        assert np.min(pc.pbc_margin(R_train, base, np.linalg.inv(base))) >= 1e-6
    lat_and_inv = None if base is None else (base, np.linalg.inv(base))
    x, gd = odesc.from_R(R_train, lat_and_inv)
    p = eng.GDMLPredict(model)
    p.set_R_desc(x)
    p.set_R_d_desc(gd)
    E, F, W = p.predict_virial()
    E0, F0 = p.predict()
    assert np.array_equal(E, E0) and np.array_equal(F, F0)
    F1, W1 = p.predict_virial(return_E=False)
    assert np.array_equal(F1, F0) and np.array_equal(W1, W)
    vcc.check_cells('train %s' % kind, model, opredict.Predictor(model), R_train, None, E, F, W)
    with pytest.raises(ValueError):
        p.predict_virial(lattice=base if base is not None else np.eye(3))


def test_train_point_sharded_one_gpu(eng):
    """TrainPointShardedPredictor.predict_virial on one GPU (one rank holds every training point, raw sums scaled
    afterwards) against the oracle, NumPy and CUDA tensors, the model's cell and one cell per geometry."""
    import torch

    from sgdml_b200 import dist as sdist

    N, base, model = _periodic('d105', 151, ecstr=True)
    op = opredict.Predictor(model)
    tp = sdist.TrainPointShardedPredictor(model, eng.GDMLPredict)
    p = eng.GDMLPredict(model)
    R = vc.queries(N, 11, 152, base)
    cells = vcc.cells_for(R, base, 153)
    for lat, cc in ((None, None), (cells, cells)):
        E, F, W = tp.predict_virial(R, lattice=lat)
        vcc.check_cells('train-point sharded numpy', model, op, R, cc, E, F, W)
        Et, Ft, Wt = tp.predict_virial(torch.from_numpy(R).cuda(), lattice=lat)
        torch.cuda.synchronize()
        assert Wt.is_cuda and Wt.shape == (11, 3, 3)
        vcc.check_cells('train-point sharded cuda', model, op, R, cc, _np(Et), _np(Ft), _np(Wt))
        Ed, Fd, Wd = p.predict_virial(R, lattice=lat)
        vcc.check_cells('unsharded', model, op, R, cc, Ed, Fd, Wd)
