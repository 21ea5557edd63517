"""Constant-pressure MD on the device (sgdml_b200_npt_*, sgdml_b200.GDMLNPTDynamics) against the NumPy restatement of
tests/npt_oracle.py, fed by sgdml_b200_predict_virial_cells on device-resident positions in the restatement's own
cells and inverses.

GPU: trajectories against the restatement (a small periodic fixture and a D > 256 periodic model), zero
compressibility against sgdml_b200_md_run, graph against plain launches and chunks, reproducibility and continuation,
isolation from the predictor's calls, bad input, the public units and stress, and the isothermal-isobaric ensemble of
an ideal gas and of a trained periodic model.  Which entry points take an NPT handle is tests/test_md_handle_kinds.py's.
"""

import ctypes

import numpy as np
import pytest

import npt_oracle
from conftest import rel_err
from md_common import md_fs_masses

pytestmark = pytest.mark.gpu


def _model(name):
    """(model dict, R0 candidates (n, 3N)): a golden periodic fixture, or 'synth_n24', a random periodic model with
    D = 276 > 256 (the GEMM-composed predictor)."""
    if name == 'synth_n24':
        from sgdml_b200 import synth

        model = synth.random_model(24, 12, np.arange(24)[None], 10.0, seed=4, alpha_scale=0.1)
        model['lattice'] = np.diag([9.0, 9.5, 10.0]) + 0.2 * np.eye(3)[[1, 2, 0]]
        return model, synth.geometries(24, 8, 5).reshape(8, -1)
    import hvp_oracle

    model, Rq, _ = hvp_oracle.fixture_model(name)
    return model, np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)


def _setup(name, n_rep=2, chunk=0, model=None):
    """(GDMLPredict, GDMLNPTDynamics in model units, R0, V0, dt, base cells L0, L0inv (n_rep, 9)): replica r's
    geometry and the model's cell scaled by 1 + 0.02 (r % 3), inverses from the model's.  The handle starts in the
    model's cell."""
    import sgdml_b200
    from sgdml_b200 import _lib

    m, Rc = _model(name)
    gp = sgdml_b200.GDMLPredict(m if model is None else model)
    N = gp.n_atoms
    masses = md_fs_masses(np.linspace(1.0, 16.0, N))
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        dyn = sgdml_b200.GDMLNPTDynamics(gp, masses, n_replicas=n_rep, E_to_eV=1.0, F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    lat, inv = gp.lat_and_inv
    sc = 1.0 + 0.02 * (np.arange(n_rep) % 3)
    L0 = lat.reshape(1, 9) * sc[:, None]
    L0inv = inv.reshape(1, 9) / sc[:, None]
    R0 = Rc[np.arange(n_rep) % Rc.shape[0]] * sc[:, None]
    _, F0 = gp.predict(R0[:1])
    s = dyn.inv_mass.repeat(3)
    dt = float(np.sqrt(2e-3 / max(np.max(np.abs(F0 * s)), 1e-300)))
    V0 = np.random.default_rng(2).standard_normal(R0.shape) * 1e-3 / dt
    return gp, dyn, R0, V0, dt, L0, L0inv


def _cell_forces(gp):
    """The restatement's force callback: sgdml_b200_predict_virial_cells on device-resident R in the given cells."""
    import torch

    from sgdml_b200 import _lib

    def forces(R, cells, cell_invs):
        Rt = torch.from_numpy(np.ascontiguousarray(R)).cuda()
        n = R.shape[0]
        E = torch.empty(n, dtype=torch.float64, device='cuda')
        F = torch.empty_like(Rt)
        W = torch.empty((n, 9), dtype=torch.float64, device='cuda')
        lat, inv = np.ascontiguousarray(cells), np.ascontiguousarray(cell_invs)
        _lib.check(_lib.lib().sgdml_b200_predict_virial_cells(gp._handle, Rt.data_ptr(), n, lat.ctypes.data,
                                                              inv.ctypes.data, E.data_ptr(), F.data_ptr(), W.data_ptr(),
                                                              _lib.current_stream()), 'predict_virial_cells')
        torch.cuda.synchronize()
        return E.cpu().numpy(), F.cpu().numpy(), W.cpu().numpy()

    return forces


def _barostat(dyn, gp, R0, V0, dt, L0, L0inv):
    """(gamma, kT, P0, beta_T, tau_p) in model units that move the cells visibly within 50 steps."""
    s = dyn.inv_mass.repeat(3)
    kT = float(np.mean(V0 * V0 / s))
    E, F, W = _cell_forces(gp)(R0, L0, L0inv)
    P = npt_oracle.pressure(npt_oracle.kinetic(V0, s), W, npt_oracle.det3(L0), np.zeros(len(R0)))
    P0 = 0.5 * float(np.mean(P)) - 0.1 * float(np.max(np.abs(P)))
    tau_p = 20.0 * dt
    beta_T = 2e-4 * tau_p / (dt * float(np.max(np.abs(P - P0))))
    return 0.1 / dt, kT, P0, beta_T, tau_p


def _same(a, b):
    return set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize('name', ['pbc_n6_m8', 'synth_n24'])
def test_matches_restatement(name):
    gp, dyn, R0, V0, dt, L0, L0inv = _setup(name)
    if name == 'synth_n24':
        assert gp.n_atoms * (gp.n_atoms - 1) // 2 > 256
    dyn._set_cells_raw(L0, L0inv)
    dyn._set_state_raw(R0, V0, step=(1 << 32) - 25)  # the counter crosses 2^32 inside the run
    args = _barostat(dyn, gp, R0, V0, dt, L0, L0inv)
    seed = (9 << 32) + 4
    fr = dyn._run_raw(50, dt, *args, seed=seed, stride=10)
    s = dyn.inv_mass.repeat(3)
    gamma, kT, P0, beta_T, tau_p = args
    fin, ref = npt_oracle.run(_cell_forces(gp), R0, V0, s, L0, L0inv, 50, dt, gamma, kT, P0, beta_T, tau_p, seed=seed,
                              step0=(1 << 32) - 25, stride=10)
    keys = ('R', 'V', 'cell', 'P', 'E_pot', 'E_kin')
    whole = max(rel_err(fr[k], ref[k]) for k in keys)
    print('%s: cell change %.3g, whole-run deviation %.3g, R bit-identical: %s'
          % (name, rel_err(ref['cell'][-1], L0), whole, np.array_equal(fr['R'], ref['R'])))
    assert rel_err(ref['cell'][-1], L0) > 1e-4  # the barostat moved the cells
    # The device's exp, log and cos may differ from NumPy's in the last bit, and so may the cell of a restarted
    # restatement (its eps recovered from the cell's volume).  pbc_n6_m8's energy, forces and virial are sums of terms
    # of both signs whose cancellation turns such a last-bit change of the cell into about 1e-11 of E_pot, of the forces
    # (and so of V, through the last half-kick) and of P within one step; the trajectory then grows it to about 1e-9
    # over these 50 steps, while the D = 276 model stays within 1e-14.  So the same run is repeated with a frame after
    # every step, which must give the same frames bit for bit, and every step is restated from the device's own frame
    # before it: R, the cell and E_kin at test_md.py's tolerance, V, E_pot and P (relative to the size of its kinetic and
    # diagonal virial terms) within 1e-9, and the whole run within 1e-8.
    dyn._set_cells_raw(L0, L0inv)
    dyn._set_state_raw(R0, V0, step=(1 << 32) - 25)
    fr1 = dyn._run_raw(50, dt, *args, seed=seed, stride=1)
    assert all(np.array_equal(fr1[k][9::10], fr[k]) for k in keys)
    V0c = npt_oracle.det3(L0)
    start = (R0, V0, np.zeros(2))
    for f in range(50):
        sfin, seg = npt_oracle.run(_cell_forces(gp), start[0], start[1], s, L0, L0inv, 1, dt, gamma, kT, P0, beta_T,
                                   tau_p, seed=seed, step0=(1 << 32) - 25 + f, stride=1, eps=start[2])
        for k in ('R', 'cell', 'E_kin'):
            assert rel_err(fr1[k][f], seg[k][0]) < 1e-11, (f, k)
        for k in ('V', 'E_pot'):
            assert rel_err(fr1[k][f], seg[k][0]) < 1e-9, (f, k)
        Wd = sfin['W'][:, [0, 4, 8]]
        scale = (2.0 * seg['E_kin'][0] + np.abs(Wd).sum(1)) / (3.0 * npt_oracle.det3(seg['cell'][0]))
        assert np.all(np.abs(fr1['P'][f] - seg['P'][0]) <= 1e-9 * scale), f
        start = (fr1['R'][f], fr1['V'][f], np.log(npt_oracle.det3(fr1['cell'][f]) / V0c))
    assert whole < 1e-8
    c = dyn._get_cells_raw()
    assert np.array_equal(c['lattice'], fr['cell'][-1])
    assert rel_err(c['lattice_inv'], npt_oracle.cells(L0, L0inv, fin['eps'])[1]) < 1e-8
    assert rel_err(c['W'], fin['W']) < 1e-8


def test_zero_compressibility_is_md_run():
    import sgdml_b200

    gp, dyn, R0, V0, dt, _, _ = _setup('pbc_n6_m8', n_rep=3)  # every cell the model's
    md = sgdml_b200.GDMLDynamics(gp, md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms)), n_replicas=3, E_to_eV=1.0,
                                 F_to_eV_Ang=1.0)
    s = dyn.inv_mass.repeat(3)
    gamma, kT = 0.1 / dt, float(np.mean(V0 * V0 / s))
    dyn._set_state_raw(R0, V0, step=11)
    md._set_state_raw(R0, V0, step=11)
    a = dyn._run_raw(30, dt, gamma, kT, 0.37, 0.0, 5.0, seed=3, stride=10)
    b = md._run_raw(30, dt, gamma, kT, seed=3, stride=10)
    for k in ('R', 'V', 'E_pot', 'E_kin'):
        assert np.array_equal(a[k], b[k]), k
    lat = gp.lat_and_inv[0].ravel()
    assert np.all(a['cell'] == lat)
    vol = npt_oracle.det3(lat)
    for f in range(a['R'].shape[0]):
        _, _, W = gp.predict_virial(a['R'][f])
        W = W.reshape(-1, 9)
        want = (2.0 * a['E_kin'][f] + ((W[:, 0] + W[:, 4]) + W[:, 8])) / (3.0 * vol)
        assert rel_err(a['P'][f], want) < 1e-13
    sa, sb = dyn._get_state_raw(), md._get_state_raw()
    assert _same(sa, sb)


def test_graph_matches_plain_launches_and_chunks(monkeypatch):
    gp, dyn, R0, V0, dt, L0, L0inv = _setup('pbc_n6_m8', n_rep=5)
    args = _barostat(dyn, gp, R0, V0, dt, L0, L0inv)

    def run(d):
        d._set_cells_raw(L0, L0inv)
        d._set_state_raw(R0, V0)
        return d._run_raw(20, dt, *args, seed=8, stride=5)

    a = run(dyn)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = run(dyn)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    _, dc, _, _, _, _, _ = _setup('pbc_n6_m8', n_rep=5, chunk=2)
    c = run(dc)
    assert _same(a, c)


def test_reproducible_and_continuable():
    gp, dyn, R0, V0, dt, L0, L0inv = _setup('pbc_n6_m8', n_rep=4)
    _, dyn2, _, _, _, _, _ = _setup('pbc_n6_m8', n_rep=4)
    args = _barostat(dyn, gp, R0, V0, dt, L0, L0inv)
    for d in (dyn, dyn2):
        d._set_cells_raw(L0, L0inv)
        d._set_state_raw(R0, V0, step=5)
    a = dyn._run_raw(40, dt, *args, seed=99, stride=5)
    b1 = dyn2._run_raw(20, dt, *args, seed=99, stride=5)
    b2 = dyn2._run_raw(20, dt, *args, seed=99, stride=5)
    assert _same(a, {k: np.concatenate([b1[k], b2[k]]) for k in a})
    assert _same(dyn._get_state_raw(), dyn2._get_state_raw()) and dyn._get_state_raw()['step'] == 45
    assert _same(dyn._get_cells_raw(), dyn2._get_cells_raw())
    dyn2._set_cells_raw(L0, L0inv)
    dyn2._set_state_raw(R0, V0, step=5)
    assert _same(a, dyn2._run_raw(40, dt, *args, seed=99, stride=5))
    dyn2._set_cells_raw(L0, L0inv)
    dyn2._set_state_raw(R0, V0, step=5)
    c = dyn2._run_raw(40, dt, *args, seed=100, stride=5)
    assert not np.array_equal(a['R'], c['R']) and not np.array_equal(a['cell'], c['cell'])


def test_isolated_from_predict_calls():
    import torch

    gp, dyn, R0, V0, dt, L0, L0inv = _setup('pbc_n6_m8', n_rep=3)
    _, ref, _, _, _, _, _ = _setup('pbc_n6_m8', n_rep=3)
    args = _barostat(dyn, gp, R0, V0, dt, L0, L0inv)
    out = []
    Rbig = np.tile(R0, (30, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((90, R0.shape[1]))
    before = gp.predict(R0), gp.predict(Rbig), gp.predict_virial(Rbig)
    for d, meddle in ((ref, False), (dyn, True)):
        d._set_cells_raw(L0, L0inv)
        d._set_state_raw(R0, V0)
        r1 = d._run_raw(10, dt, *args, seed=2, stride=5)
        if meddle:
            gp.predict(Rbig)
            gp.predict_hvp(Rbig, np.ones_like(Rbig))
            gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (90, 1, 1)))
        r2 = d._run_raw(10, dt, *args, seed=2, stride=5)
        out.append((r1, r2, d._get_state_raw(), d._get_cells_raw()))
    assert all(_same(x, y) for x, y in zip(out[0], out[1]))
    after = gp.predict(R0), gp.predict(Rbig), gp.predict_virial(Rbig)
    for x, y in zip(before, after):
        assert all(np.array_equal(u, v) for u, v in zip(x, y))


def test_handle_kind_rules_and_bad_input():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, dyn, R0, V0, dt, L0, L0inv = _setup('pbc_n6_m8', n_rep=3)
    L = _lib.lib()
    st = _lib.current_stream()
    masses = md_fs_masses(np.linspace(1.0, 16.0, gp.n_atoms))
    inv_mass = dyn.inv_mass
    h = ctypes.c_void_p()
    # creation: singular, non-finite, missing cells
    for lat in (np.zeros((3, 9)), np.where(np.arange(27).reshape(3, 9) == 4, np.nan, L0)):
        assert L.sgdml_b200_npt_create(ctypes.byref(h), gp._handle, 3, inv_mass.ctypes.data, lat.ctypes.data,
                                       L0inv.ctypes.data) <= -1000 and not h.value
    assert L.sgdml_b200_npt_create(ctypes.byref(h), gp._handle, 3, inv_mass.ctypes.data, None, None) <= -1000
    with pytest.raises(_lib.EngineError):
        dyn._run_raw(10, dt, 0.0, 0.0, 0.0, 0.0, 1.0)  # no state yet
    dyn._set_cells_raw(L0, L0inv)
    dyn._set_state_raw(R0, V0, step=7)
    # bad runs and cells change nothing (which handles npt_* take: tests/test_md_handle_kinds.py)
    H = dyn._handle
    before = dyn._get_state_raw(), dyn._get_cells_raw()
    good = dict(n_steps=10, dt=dt, gamma=1.0, kT=1e-3, P0=0.1, beta_T=1e-3, tau_p=1.0, stride=0)
    for bad in (dict(P0=np.nan), dict(P0=np.inf), dict(beta_T=-1e-3), dict(beta_T=np.nan), dict(tau_p=0.0),
                dict(tau_p=-1.0), dict(tau_p=np.inf), dict(gamma=0.0), dict(stride=3), dict(dt=0.0), dict(n_steps=-1),
                dict(kT=-1.0)):
        kw = dict(good, **bad)
        out = {k: np.full((4, 3, 18), 1.5) for k in ('R', 'cell')}
        rc = L.sgdml_b200_npt_run(H, kw['n_steps'], kw['dt'], kw['gamma'], kw['kT'], kw['P0'], kw['beta_T'],
                                  kw['tau_p'], 0, kw['stride'], out['R'].ctypes.data, None, None, None,
                                  out['cell'].ctypes.data, None, st)
        assert rc <= -1000, bad
        assert np.all(out['R'] == 1.5) and np.all(out['cell'] == 1.5)
    for lat, inv in ((np.zeros_like(L0), L0inv), (L0, np.full_like(L0inv, np.inf)), (L0[:, ::-1] * 0.0 + 1.0, L0inv)):
        assert L.sgdml_b200_npt_set_cells(H, np.ascontiguousarray(lat).ctypes.data,
                                          np.ascontiguousarray(inv).ctypes.data, st) <= -1000
    after = dyn._get_state_raw(), dyn._get_cells_raw()
    assert all(_same(x, y) for x, y in zip(before, after))
    with pytest.raises(ValueError):
        sgdml_b200.GDMLNPTDynamics(gp, masses, cells=np.eye(3)[:2], n_replicas=3)
    from sgdml_b200 import synth

    free = synth.random_model(5, 4, np.arange(5)[None], 10.0)
    with pytest.raises(ValueError):
        sgdml_b200.GDMLNPTDynamics(free, np.ones(5))


def test_public_units():
    """GDMLNPTDynamics in eV / Angstrom / fs with a kcal/mol model: cells as rows in Angstrom, pressure in eV/A^3 and
    compressibility in A^3/eV convert to the engine's model units, and the stress is the calculator's."""
    import torch

    import sgdml_b200
    from sgdml_b200 import md
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc, SGDMLCalculatorCore

    model, Rc = _model('pbc_n6_m8')
    masses = np.linspace(1.0, 16.0, 6)
    cells = np.stack([model['lattice'].T, 1.03 * model['lattice'].T])  # rows, Angstrom (Ang_to_R = 1 here)
    d = sgdml_b200.GDMLNPTDynamics(model, masses, cells=cells, n_replicas=2)
    assert d.Ang_to_R == 1.0
    raw = d._get_cells_raw()
    assert np.array_equal(raw['lattice'], np.ascontiguousarray(cells.swapaxes(1, 2)).reshape(2, 9))
    assert np.array_equal(raw['lattice_inv'], np.linalg.inv(cells.swapaxes(1, 2)).reshape(2, 9))
    R0 = Rc[:2].reshape(2, 6, 3)
    V0 = 1e-3 * np.random.default_rng(0).standard_normal(R0.shape)
    T, fric, p, comp, taup = 300.0, 0.01, 0.002, 0.5, 50.0
    d.set_state(R0, V0)
    out = d.run(20, 0.5, T, fric, p, comp, taup, seed=1, stride=10)
    d2 = sgdml_b200.GDMLNPTDynamics(d.gdml_predict, masses, cells=cells, n_replicas=2)
    d2._set_state_raw(R0.reshape(2, -1), V0.reshape(2, -1))
    f = d2._run_raw(20, 0.5, fric, md.KB_EV * T / kc, p / kc, comp * kc, taup, 1, 10)
    assert np.array_equal(out['positions'], f['R'].reshape(2, 2, 6, 3))
    assert np.array_equal(out['cells'], f['cell'].reshape(2, 2, 3, 3).swapaxes(-1, -2))
    assert np.allclose(out['pressure'], f['P'] * kc, rtol=1e-15, atol=0)
    assert np.allclose(out['volume'], np.abs(np.linalg.det(out['cells'])), rtol=1e-13, atol=0)
    assert np.allclose(out['potential_energy'], f['E_pot'] * kc, rtol=1e-15, atol=0)
    # pressure of the frame against the stress: P = (2 E_kin - tr(stress) V) / 3V
    st = d.get_state()
    assert st['cells'].shape == (2, 3, 3) and st['stress'].shape == (2, 6)
    calc = SGDMLCalculatorCore()
    calc._setup(model, kc, kc)
    for r in range(2):
        want = calc.compute(st['positions'][r], cell=st['cells'][r], stress=True)['stress']
        assert rel_err(st['stress'][r], want) < 1e-12
    P_state = (2.0 * out['kinetic_energy'][-1] - st['stress'][:, :3].sum(1) * out['volume'][-1]) / (3.0 * out['volume'][-1])
    assert rel_err(out['pressure'][-1], P_state) < 1e-10
    # set_cells (rows, Angstrom) and CUDA tensors in -> CUDA tensors out
    d.set_cells(torch.from_numpy(cells[0]))
    assert np.array_equal(d._get_cells_raw()['lattice'], np.tile(cells[0].T.ravel(), (2, 1)))
    d.set_cells(cells)
    d.set_state(torch.from_numpy(R0).cuda(), torch.from_numpy(V0).cuda())
    t = d.run(20, 0.5, T, fric, p, comp, taup, seed=1, stride=10)
    assert t['cells'].is_cuda and np.array_equal(t['cells'].cpu().numpy(), out['cells'])
    assert np.array_equal(t['positions'].cpu().numpy(), out['positions'])
    ts = d.get_state()
    assert ts['stress'].is_cuda and rel_err(ts['stress'].cpu().numpy(), st['stress']) < 1e-14


def _mean_se(x, n_blocks=20):
    b = x.mean(1)[: len(x) // n_blocks * n_blocks].reshape(n_blocks, -1).mean(1)
    return float(b.mean()), float(b.std(ddof=1) / np.sqrt(n_blocks))


def test_ideal_gas_ensemble():
    """pbc_n6_m8 with zero coefficients (F = W = 0): <V> = (N + 1) kT / P0 within 4 standard errors, and N kT / P0,
    (N + 2) kT / P0 outside; the parameters of tests/test_npt_oracle.py::test_ideal_gas_volume."""
    model, _ = _model('pbc_n6_m8')
    model = dict(model, alphas_F=np.zeros_like(model['alphas_F']), R_d_desc_alpha=np.zeros_like(model['R_d_desc_alpha']))
    gp, dyn, R0, _, _, _, _ = _setup('pbc_n6_m8', n_rep=256, model=model)
    N = gp.n_atoms
    a = 7.0 ** (1.0 / 3.0)
    dyn._set_cells_raw(np.tile((a * np.eye(3)).ravel(), (256, 1)), np.tile((np.eye(3) / a).ravel(), (256, 1)))
    V0 = np.random.default_rng(0).standard_normal(R0.shape) * np.sqrt(1.0 / np.linspace(1.0, 16.0, N).repeat(3))
    dyn._set_state_raw(R0, V0)
    args = (0.02, 1.0, 1.0, 1.0, 1.0, 1.0)  # dt, gamma, kT, P0, beta_T, tau_p
    dyn._run_raw(500, *args, seed=7, frames=())
    fr = dyn._run_raw(4000, *args, seed=7, stride=10, frames=('cell',))
    vol = npt_oracle.det3(fr['cell'])
    m, se = _mean_se(vol)
    print('ideal gas on the device: <V> = %.4f +- %.4f, exact %d' % (m, se, N + 1))
    assert abs(m - (N + 1)) < 4.0 * se
    assert abs(m - N) > 4.0 * se and abs(m - (N + 2)) > 4.0 * se


# O(dt) allowance of <V (P0 - P_int)> in units of kT: the restatement's volume-only energy
# (tests/test_npt_oracle.py::test_volume_energy_against_quadrature, c_a times the volume stiffness about 0.02 per step)
# stays within 0.04 kT of kT; the run below keeps that product below 0.02.
_VIRIAL_ALLOWANCE = 0.1


def test_trained_periodic_ensemble():
    """pbc_n6_m8 in cells three times its own: <V (P0 - P_int)> = kT, which holds only when the virial and the kinetic
    pressure enter P_int correctly (without the virial the molecule's atoms would count as N free particles)."""
    gp, dyn, R0, V0, dt, _, _ = _setup('pbc_n6_m8', n_rep=128)
    s = dyn.inv_mass.repeat(3)
    lat, inv = gp.lat_and_inv
    vol0 = 27.0 * npt_oracle.det3(lat.ravel())
    # cells three times the model's: a proper ensemble at any P0 > 0, whatever the energy does at large volumes
    dyn._set_cells_raw(np.tile(3.0 * lat.ravel(), (128, 1)), np.tile(inv.ravel() / 3.0, (128, 1)))
    # test_md.py's equipartition setting: kT well above the model's small thermal energy, half the step, strong coupling
    kT = 30.0 * float(np.mean(V0 * V0 / s))
    dt = 0.5 * dt
    gamma = 0.5 / dt
    V = np.random.default_rng(3).standard_normal(R0.shape) * np.sqrt(kT * s)
    dyn._set_state_raw(R0, V)
    # P0 = 2 kT / V_start: the mean volume of one free particle at V_start (the molecule's centre of mass), and the
    # volume stiffness dP_int/d(eps) about P0, so that c_a times it is 0.01 per step
    P0 = 2.0 * kT / vol0
    tau_p = 1.0
    beta_T = 0.01 * tau_p / (dt * P0)
    print('kT %.4g, P0 %.4g, beta_T %.4g' % (kT, P0, beta_T))
    dyn._run_raw(1000, dt, gamma, kT, P0, beta_T, tau_p, seed=2, frames=())
    fr = dyn._run_raw(6000, dt, gamma, kT, P0, beta_T, tau_p, seed=2, stride=5, frames=('cell', 'P'))
    vol = npt_oracle.det3(fr['cell'])
    m, se = _mean_se(vol * (P0 - fr['P']) / kT)
    print('trained periodic model: <V (P0 - P_int)> / kT = %.4f +- %.4f, <V> / V_start = %.4f'
          % (m, se, vol.mean() / vol0))
    assert np.all(np.isfinite(vol)) and np.all(np.isfinite(fr['P']))
    assert abs(m - 1.0) < 4.0 * se + _VIRIAL_ALLOWANCE
