"""The predictor at the batch sizes it is benchmarked at: several chunks per call, the pipelined host-I/O path on two
workspace slots, small tail chunks inside bulk calls, and -- through the chunk-size test hook
sgdml_b200_set_predict_chunk -- the same paths at small batches, against the oracle with the componentwise bound of
tests/predict_checks.py.

Every model is built with the oracle's descriptor code, so that the reference shares no GPU code.  Output buffers
passed with out= are filled with NaN first, and two calls on one handle always see different inputs, so that a
missing copy or a stale workspace slot cannot pass.  The engine's launch counters (not its profiler, which switches the
pipeline and the graph path off) confirm that each call ran the plan chunk_plan predicts."""

import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import predict_checks as pc  # noqa: E402
from conftest import rel_err  # noqa: E402
from oracle import assemble as oassemble  # noqa: E402
from oracle import desc as odesc  # noqa: E402
from oracle import predict as opredict  # noqa: E402


@pytest.fixture(scope='module')
def eng():
    import sgdml_b200
    from sgdml_b200 import _lib

    _lib.require_gpu()
    return sgdml_b200


def _model(N, M, perms, sig, r0=None, seed=0):
    """Random-coefficient model of the benchmark's recipe (training geometries seed 0, coefficients seed 99), with
    std and c away from 1 and 0 so that the output scaling is checked too."""
    from sgdml_b200 import synth

    R = synth.geometries(N, M, seed, r0=r0).reshape(M, -1)
    alphas = np.random.default_rng(seed + 99).standard_normal(M * 3 * N)
    x, g = odesc.from_R(R)
    perms = np.asarray(perms, dtype=np.int64)
    model = {
        'type': 'm',
        'z': np.ones(N, dtype=np.int64),
        'R_desc': np.ascontiguousarray(x.T),
        'R_d_desc_alpha': odesc.d_desc_dot_vec(g, alphas.reshape(M, -1)),
        'alphas_F': alphas,
        'c': 0.37,
        'std': 1.7,
        'sig': sig,
        'lam': 1e-10,
        'perms': perms,
        'tril_perms_lin': odesc.tril_perms_lin(perms),
        'use_E': True,
    }
    return model, x, g


def _main_launches():
    from sgdml_b200 import _lib

    return _lib.profile_snapshot()['predict_main'][2]


@contextlib.contextmanager
def _chunk_cap(n):
    from sgdml_b200 import _lib

    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(int(n)), 'set_predict_chunk')
    try:
        yield
    finally:
        _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(0), 'set_predict_chunk')


def _plan(model, B, host_io, cap=0, train=False):
    N = int(np.asarray(model['z']).shape[0])
    ly = pc.layout(N, model['R_desc'].shape[1])
    return pc.chunk_plan(ly.D, ly.DP, ly.Mpad, len(model['perms']), ly.large, B, host_io, cap=cap, train=train)


def _run(p, R, plan, **kw):
    """p.predict(R, **kw), asserting that it took `plan` (launch count of the main predictor kernels)."""
    import torch

    n0 = _main_launches()
    out = p.predict(R, **kw)
    torch.cuda.synchronize()
    got = _main_launches() - n0
    assert got == plan.main_launches, 'main-kernel launches %d, plan %d (%d chunks)' % (got, plan.main_launches, len(plan.chunks))
    return out


def _np(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def _nan_out(B, dim_i, pinned=False, numpy=False):
    import torch

    if numpy:
        return np.full(B, np.nan), np.full((B, dim_i), np.nan)
    E = torch.full((B,), float('nan'), dtype=torch.float64)
    F = torch.full((B, dim_i), float('nan'), dtype=torch.float64)
    return (E.pin_memory(), F.pin_memory()) if pinned else (E, F)


def _check(tag, model, op, R, rows, E, F):
    """check_predict on `rows` of (E, F) against the oracle; prints the observed max |err| / scale against tau."""
    rows = np.asarray(sorted(set(int(r) for r in rows)))
    Rr = R[rows]
    E_ref, F_ref = op.predict(Rr)
    scale = pc.predict_abs_scale(model, Rr, oracle=op)
    M, D = model['R_desc'].shape[1], model['R_desc'].shape[0]
    k = pc.n_terms(M, op.n_perms, D)
    rF, rE = pc.check_predict(None if E is None else _np(E)[rows], _np(F)[rows], E_ref, F_ref, scale, k, what=tag)
    print('\n[predict bound] %s: %d rows, max|err|/scale F %.2e E %s, tau %.2e' % (
        tag, len(rows), rF, 'n/a' if rE is None else '%.2e' % rE, pc.tau(k)))
    assert rF <= pc.tau(k) / 10 and (rE is None or rE <= pc.tau(k) / 10), 'less than 10x margin below tau'


def _sample(B, n, seed):
    return np.random.default_rng(seed).choice(B, size=min(n, B), replace=False)


# --------------------------------------------------------------------------- BASELINE config 2 (aspirin)
def test_bench_config2_four_routes(eng):
    """aspirin, M = 1000, S = 6, sigma 20, B = 65 536 (the benchmark's batch and query seed) through the four routes
    the benchmark times: all four bit-identical, chunk edges and 64 seeded rows within the bound of the oracle."""
    import torch
    from sgdml_b200 import synth

    perms, r0 = synth.config_perms_and_r0('aspirin')
    N, M, B = 21, 1000, 65536
    model, _, _ = _model(N, M, perms, 20, r0=r0)
    dim_i = 3 * N
    Rq = synth.geometries(N, B, 1, r0=r0).reshape(B, -1)
    Rx = synth.geometries(N, B, 7, r0=r0).reshape(B, -1)  # other inputs, run before each route on the same handle
    p = eng.GDMLPredict(model)
    dev, host = _plan(model, B, False), _plan(model, B, True)
    assert len(dev.chunks) == 3 and host.pipelined and host.slots == [0, 1, 0, 1]

    # 1. CUDA tensors in and out
    p.predict(torch.from_numpy(Rx).cuda())
    E1, F1 = _run(p, torch.from_numpy(Rq).cuda(), dev)
    E1, F1 = E1.cpu().numpy(), F1.cpu().numpy()
    # 2. pinned tensors with out=
    R_pin = torch.from_numpy(Rq).pin_memory()
    p.predict(torch.from_numpy(Rx).pin_memory(), out=_nan_out(B, dim_i, pinned=True))
    out2 = _nan_out(B, dim_i, pinned=True)
    E2, F2 = _run(p, R_pin, host, out=out2)
    assert E2 is out2[0] and F2 is out2[1]
    # 3. pageable NumPy, new arrays out
    p.predict(Rx)
    E3, F3 = _run(p, Rq, host)
    # 4. NumPy, forces only, into NaN-filled out=
    p.predict(Rx, return_E=False)
    out4 = _nan_out(B, dim_i, numpy=True)
    (F4,) = _run(p, Rq, host, return_E=False, out=out4)
    assert np.all(np.isnan(out4[0]))  # the energy buffer is not touched

    for E, F in ((E2.numpy(), F2.numpy()), (E3, F3), (None, F4)):
        assert np.array_equal(F, F1)
        if E is not None:
            assert np.array_equal(E, E1)
    op = opredict.Predictor(model)
    rows = pc.edge_rows(dev) + pc.edge_rows(host) + list(_sample(B, 64, 2024))
    _check('aspirin B=65536', model, op, Rq, rows, E1, F1)


# --------------------------------------------------------------------------- BASELINE config 1 (ethanol)
@pytest.fixture(scope='module')
def ethanol(eng):
    from sgdml_b200 import synth

    perms, r0 = synth.config_perms_and_r0('ethanol')
    model, _, _ = _model(9, 200, perms, 20, r0=r0)
    return model, opredict.Predictor(model), r0


def test_ethanol_bench_batch_device_and_host(eng, ethanol):
    import torch
    from sgdml_b200 import synth

    model, op, r0 = ethanol
    B = 65536
    Rq = synth.geometries(9, B, 1, r0=r0).reshape(B, -1)
    p = eng.GDMLPredict(model)
    dev, host = _plan(model, B, False), _plan(model, B, True)
    assert len(dev.chunks) == 1 and len(host.chunks) == 4
    E1, F1 = _run(p, torch.from_numpy(Rq).cuda(), dev)
    p.predict(synth.geometries(9, B, 8, r0=r0).reshape(B, -1))
    out = _nan_out(B, 27, numpy=True)
    E2, F2 = _run(p, Rq, host, out=out)
    assert np.array_equal(E2, E1.cpu().numpy()) and np.array_equal(F2, F1.cpu().numpy())
    _check('ethanol B=65536', model, op, Rq, pc.edge_rows(dev) + pc.edge_rows(host) + list(_sample(B, 64, 3)), E2, F2)


def test_ethanol_tail_chunk(eng, ethanol):
    """3 x 65 536 + 3 on the device: the 3-geometry tail splits the sweep over the training points and runs
    k_predict_finish_small on a workspace sized for 65 536 queries."""
    import torch
    from sgdml_b200 import synth

    model, op, r0 = ethanol
    B = 3 * 65536 + 3
    Rq = synth.geometries(9, B, 11, r0=r0).reshape(B, -1)
    p = eng.GDMLPredict(model)
    plan = _plan(model, B, False)
    assert plan.chunks[-1] == (196608, 196611)
    p.predict(torch.from_numpy(synth.geometries(9, B, 12, r0=r0).reshape(B, -1)).cuda())
    E, F = _run(p, torch.from_numpy(Rq).cuda(), plan)
    _check('ethanol B=196611', model, op, Rq, pc.edge_rows(plan) + [B - 3, B - 2, B - 1], E, F)


@pytest.mark.parametrize('B', [16, 17, 4095, 4096, 4097])
def test_ethanol_host_thresholds(eng, ethanol, B):
    """Host buffers at the graph-replay (16 / 17) and pipeline (4095 / 4096) boundaries: every row against the oracle.
    The first call at a batch size captures the graph; the checked call is a replay on other inputs."""
    from sgdml_b200 import synth

    model, op, r0 = ethanol
    Rq = synth.geometries(9, B, 20 + B, r0=r0).reshape(B, -1)
    p = eng.GDMLPredict(model)
    p.predict(synth.geometries(9, B, 21 + B, r0=r0).reshape(B, -1))
    out = _nan_out(B, 27, numpy=True)
    E, F = _run(p, Rq, _plan(model, B, True), out=out)
    _check('ethanol host B=%d' % B, model, op, Rq, range(B), E, F)


# --------------------------------------------------------------------------- config 3 shape (D = 861, GEMM-composed)
def _slices_equal(p, Rd, F_bulk, bounds):
    import torch

    parts = [p.predict(Rd[lo:hi])[1] for lo, hi in bounds]
    torch.cuda.synchronize()
    return torch.equal(torch.cat(parts), F_bulk)


def test_config3_bulk_equals_slices(eng):
    """N = 42, S = 243, sigma 50, M = 2000, B = 4096 (8 chunks of up to 552): the GEMM-composed path has no
    batch-dependent split, so the bulk call is bit-identical to chunk-aligned and to misaligned slices -- in FP64 and
    on 5 int8 slices, which agree with FP64 to 1e-8.  (At this M the oracle would need ~3 GB of permuted caches per
    query: the values are checked against it at reduced M below.)"""
    import torch
    from sgdml_b200 import synth

    perms, r0 = synth.config_perms_and_r0('ac-ala3-nhme')
    N, M, B = 42, 2000, 4096
    model, _, _ = _model(N, M, perms, 50, r0=r0)
    Rd = torch.from_numpy(synth.geometries(N, B, 1, r0=r0).reshape(B, -1)).cuda()
    p = eng.GDMLPredict(model)
    plan = _plan(model, B, False)
    assert len(plan.chunks) == 8
    misaligned = [(lo, min(lo + 100, B)) for lo in range(0, B, 100)]
    _, F64 = _run(p, Rd, plan)
    F64 = F64.clone()
    assert _slices_equal(p, Rd, F64, plan.chunks)
    assert _slices_equal(p, Rd, F64, misaligned)
    p.set_contraction_slices(5)
    _, F5 = _run(p, Rd, plan)
    F5 = F5.clone()
    assert _slices_equal(p, Rd, F5, plan.chunks)
    assert _slices_equal(p, Rd, F5, misaligned)
    assert rel_err(F5.cpu().numpy(), F64.cpu().numpy()) < 1e-8


def test_config3_shape_reduced_m_capped(eng):
    """The same shape at M = 100 (the last 8-point tile half padded) with at most 7 queries per chunk: every row
    against the oracle."""
    import torch
    from sgdml_b200 import synth

    perms, r0 = synth.config_perms_and_r0('ac-ala3-nhme')
    N, M, B = 42, 100, 12
    model, _, _ = _model(N, M, perms, 50, r0=r0)
    Rq = synth.geometries(N, B, 1, r0=r0).reshape(B, -1)
    with _chunk_cap(7):
        p = eng.GDMLPredict(model)
        plan = _plan(model, B, False, cap=7)
        assert plan.chunks == [(0, 7), (7, 12)]
        p.predict(torch.from_numpy(synth.geometries(N, B, 2, r0=r0).reshape(B, -1)).cuda())
        E, F = _run(p, torch.from_numpy(Rq).cuda(), plan)
    _check('ac-ala3 shape M=100 cap 7', model, opredict.Predictor(model), Rq, range(B), E, F)


# --------------------------------------------------------------------------- predict_train / K.v
def _c60_model(M, seed=0):
    from sgdml_b200 import synth

    perms, r0 = synth.config_perms_and_r0('c60')
    return _model(60, M, perms, 50, r0=r0, seed=seed)


def test_kv_c60_multi_chunk(eng):
    """c60 (I_h, S = 120), M = 3000: K.v runs as 4 chunks of 745 training points and a tail of 20, bit-identical to
    single-chunk calls, in FP64 and on 5 int8 slices."""
    model, x, g = _c60_model(3000)
    M = 3000
    p = eng.GDMLPredict(model)
    p.set_R_desc(x)
    p.set_R_d_desc(g)
    p.set_alphas(np.random.default_rng(5).standard_normal(M * 180))
    plan = _plan(model, M, False, train=True)
    assert len(plan.chunks) == 5 and plan.chunks[-1] == (2980, 3000)
    for slices in (0, 5):
        p.set_contraction_slices(slices)
        n0 = _main_launches()
        full = p.kmatvec_train(0, M).copy()
        assert _main_launches() - n0 == plan.main_launches
        parts = np.concatenate([p.kmatvec_train(lo, hi) for lo, hi in plan.chunks])
        assert np.array_equal(full, parts), slices
        assert np.all(np.isfinite(full))


def test_kv_and_training_predictions_capped(eng):
    """c60 at M = 5 with 2 training points per chunk: predict() with R=None and K.v over odd row ranges against the
    oracle's kernel matrix."""
    M = 5
    model, x, g = _c60_model(M, seed=3)
    v = np.random.default_rng(6).standard_normal(M * 180)
    K = oassemble.assemble(x, g, model['tril_perms_lin'], 50)
    with _chunk_cap(2):
        p = eng.GDMLPredict(model)
        p.set_R_desc(x)
        p.set_R_d_desc(g)
        n0 = _main_launches()
        E, F = p.predict()
        assert _main_launches() - n0 == _plan(model, M, False, cap=2, train=True).main_launches == 6
        p.set_alphas(v)
        for lo, hi in ((1, 4), (3, 5), (0, 5)):
            plan = _plan(model, hi - lo, False, cap=2, train=True)
            out = np.full((hi - lo, 180), np.nan)
            n0 = _main_launches()
            p.kmatvec_train(lo, hi, out=out)
            assert _main_launches() - n0 == plan.main_launches
            assert rel_err(out.ravel(), K[lo * 180 : hi * 180] @ v) < 1e-10, (lo, hi)
    op = opredict.Predictor(model)
    op.set_R_desc(x)
    op.set_R_d_desc(g)
    E_ref, F_ref = op.predict()
    scale = pc.predict_abs_scale(model, oracle=op, R_desc=x, R_d_desc=g)
    rF, rE = pc.check_predict(E, F, E_ref, F_ref, scale, pc.n_terms(M, 120, 1770), what='c60 R=None')
    assert rF <= pc.tau(pc.n_terms(M, 120, 1770)) / 10


# --------------------------------------------------------------------------- cap sweep
SWEEP_SHAPES = {
    # name: (N, M, rotors, swaps, sig); M is not a multiple of the training tile BM
    'ethanol': (9, 200, 1, 1, 20),  # BM 32
    'aspirin': (21, 40, 1, 1, 20),  # BM 16
    'd276': (24, 29, 1, 1, 30),  # D > 256, BM 8
}
SWEEP_B = (1, 7, 23, 4097)


@pytest.fixture(scope='module', params=sorted(SWEEP_SHAPES))
def sweep_case(request, eng):
    from sgdml_b200 import synth

    N, M, rot, swap, sig = SWEEP_SHAPES[request.param]
    assert M % pc.layout(N, M).BM != 0
    model, _, _ = _model(N, M, synth.rotor_swap_group(N, rot, swap), sig, seed=N)
    op = opredict.Predictor(model)
    Rs = {B: synth.geometries(N, B, 40 + B).reshape(B, -1) for B in SWEEP_B}
    refs = {B: op.predict(Rs[B]) for B in SWEEP_B}
    scales = {B: pc.predict_abs_scale(model, Rs[B], oracle=op) for B in SWEEP_B}
    return request.param, model, Rs, refs, scales


@pytest.mark.parametrize('cap', [1, 2, 5, 7])
def test_cap_sweep(eng, sweep_case, cap):
    """B = 1, 7, 23 from device tensors and B = 4097 from NumPy arrays (a pipeline of hundreds of chunks alternating
    between the two slots), at most `cap` queries per chunk: every row against the oracle."""
    import torch

    name, model, Rs, refs, scales = sweep_case
    M, D = model['R_desc'].shape[1], model['R_desc'].shape[0]
    k = pc.n_terms(M, len(model['perms']), D)
    worst = 0.0
    with _chunk_cap(cap):
        p = eng.GDMLPredict(model)
        for B in SWEEP_B:
            host = B > 1000
            plan = _plan(model, B, host, cap=cap)
            assert len(plan.chunks) == -(-B // cap) and plan.pipelined == host
            if host:
                out = _nan_out(B, Rs[B].shape[1], numpy=True)
                E, F = _run(p, Rs[B], plan, out=out)
            else:
                E, F = _run(p, torch.from_numpy(Rs[B]).cuda(), plan)
                E, F = E.cpu().numpy(), F.cpu().numpy()
            rF, rE = pc.check_predict(E, F, refs[B][0], refs[B][1], scales[B], k, what='%s cap %d B %d' % (name, cap, B))
            worst = max(worst, rF, rE)
    print('\n[predict bound] sweep %s cap %d: max|err|/scale %.2e, tau %.2e' % (name, cap, worst, pc.tau(k)))
    assert worst <= pc.tau(k) / 10
