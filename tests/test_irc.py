"""The reaction path on the device (sgdml_b200_irc_rk4, sgdml_b200.GDMLIRC) against the NumPy restatement of
tests/irc_oracle.py driven by GDMLPredict.predict: every predictor form, int8 slices, all three end codes in one call,
graph against plain launches, block lengths, chunks that split a pair, a pair alone and among many, isolation from the
predictor's own calls and from other handles, host, device and NULL outputs, public units, argument errors and handle
kinds; and the two minima a saddle connects on the double-well hinge model of tests/test_neb.py, trained in the test.
"""

import ctypes

import numpy as np
import pytest

import irc_oracle
from conftest import rel_err
from md_common import FIXTURES_MD, _cuda_forces, md_fs_masses
from relax_oracle import atom_max2

pytestmark = pytest.mark.gpu

_KEYS = ('R', 'F', 'E', 'R_path', 'E_path', 'n_points', 'end', 'fmax')


def _masses(N):
    """masses for which GDMLIRC in model units has the inverse masses 1 / m, m = 1, 2, 3, 1, ..."""
    return md_fs_masses(1.0 + np.arange(N) % 3)


def _setup(name, n_saddles=2, chunk=0, slices=0):
    """(GDMLPredict, GDMLIRC in model units with the inverse masses 1 / m, m = 1, 2, 3, 1, ..., saddles (n_saddles,
    3N), modes (n_saddles, 3N), step).  The saddles are the fixture's query geometries, the modes seeded normals."""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    gp = sgdml_b200.GDMLPredict(model)
    if slices:
        gp.set_contraction_slices(slices)
    N = gp.n_atoms
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        irc = sgdml_b200.GDMLIRC(gp, _masses(N), n_saddles, E_to_eV=1.0, F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    X = np.asarray(Rq, dtype=np.float64).reshape(-1, 3 * N)
    R0 = X[np.arange(n_saddles) % len(X)] + 1e-2 * np.random.default_rng(1).standard_normal((n_saddles, 3 * N))
    modes = np.random.default_rng(2).standard_normal((n_saddles, 3 * N))
    _, F0 = gp.predict(R0)
    h = 2e-3 / max(float(np.max(np.abs(F0))), 1.0) ** 0.5  # a small fraction of the distance to the nearby minima
    return gp, irc, R0, modes, h


def _device(irc, R0, modes, mp, h, fmax):
    if R0 is not None:
        irc._set_state_raw(np.repeat(R0, 2, axis=0))
    Rp, Ep, n, end, fm = irc._irc_raw(modes, mp, h, fmax)
    st = irc._get_state_raw()
    return {'R': st['R'], 'F': st['F'], 'E': st['E_pot'], 'V': st['V'], 'step': st['step'], 'R_path': Rp,
            'E_path': Ep, 'n_points': n, 'end': end, 'fmax': fm}


def _oracle(gp, irc, R0, modes, mp, h, fmax):
    forces = _cuda_forces(gp)
    E0, F0 = forces(R0)
    return irc_oracle.irc(forces, R0, E0, F0, modes, np.repeat(irc.inv_mass, 3), mp, h, fmax)


def _same(a, b, keys=_KEYS):
    return all(np.array_equal(a[k], b[k], equal_nan=True) for k in keys)


def _check_against(dev, ref):
    bad = [k for k in _KEYS if not np.array_equal(dev[k], ref[k], equal_nan=True)]
    assert not bad, (bad, [rel_err(np.nan_to_num(dev[k]), np.nan_to_num(ref[k])) for k in bad])
    assert np.all(dev['V'] == 0.0) and dev['step'] == 0
    for b in range(len(dev['n_points'])):  # NaN past n_points, the branch end in the state
        n = dev['n_points'][b]
        assert np.all(np.isnan(dev['R_path'][b, n:])) and np.all(np.isnan(dev['E_path'][b, n:]))
        assert np.all(np.isfinite(dev['E_path'][b, :n]))
        assert np.array_equal(dev['R'][b], dev['R_path'][b, n - 1]) and dev['E'][b] == dev['E_path'][b, n - 1]


# ---------------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_matches_restatement(name):
    gp, irc, R0, modes, h = _setup(name)
    dev = _device(irc, R0, modes, 10, h, 0.0)
    ref = _oracle(gp, irc, R0, modes, 10, h, 0.0)
    print('%s: points %s, end codes %s' % (name, dev['n_points'].tolist(), dev['end'].tolist()))
    _check_against(dev, ref)
    assert dev['n_points'].max() == 10  # a branch ran to the end


def test_int8_slices():
    gp, irc, R0, modes, h = _setup('big_n100_m2_s12', slices=6)
    _check_against(_device(irc, R0, modes, 10, h, 0.0), _oracle(gp, irc, R0, modes, 10, h, 0.0))


def test_all_three_end_codes_in_one_call():
    """Six pairs from non-stationary starts: a branch whose first point rises ends at once (2); fmax between the
    smallest max_a |F_a| the descending branches reach ends some of them by force (1) and leaves others to run to
    max_points (3)."""
    gp, irc, R0, modes, h = _setup('n9_m16_s6', n_saddles=6)
    mp = 12
    probe = _oracle(gp, irc, R0, modes, mp, h, 0.0)
    full = np.flatnonzero(probe['n_points'] == mp)
    _, Fp = gp.predict(probe['R_path'][full, 1:].reshape(-1, probe['R_path'].shape[-1]))
    low = np.sqrt(atom_max2(Fp)).reshape(len(full), mp - 1).min(1)
    assert len(full) >= 2 and low.min() < low.max()
    fmax = float(np.sqrt(low.min() * low.max()))
    dev = _device(irc, R0, modes, mp, h, fmax)
    ref = _oracle(gp, irc, R0, modes, mp, h, fmax)
    print('fmax %.6g: points %s, end codes %s' % (fmax, dev['n_points'].tolist(), dev['end'].tolist()))
    _check_against(dev, ref)
    assert set(dev['end'].tolist()) == {1, 2, 3}
    assert np.all(dev['fmax'][dev['end'] == 1] < fmax)


# ---------------------------------------------------------------------------------------------------- bitwise equalities
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12', 'pbc_n6_m8'])
def test_graph_blocks_and_chunks(name, monkeypatch):
    from sgdml_b200 import _lib

    gp, irc, R0, modes, h = _setup(name, n_saddles=3)
    a = _device(irc, R0, modes, 9, h, 0.0)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _device(irc, R0, modes, 9, h, 0.0)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    for block in (1, 7, 1000):
        _lib.check(_lib.lib().sgdml_b200_set_relax_block(block), 'set_relax_block')
        try:
            c = _device(irc, R0, modes, 9, h, 0.0)
        finally:
            _lib.lib().sgdml_b200_set_relax_block(0)
        assert _same(a, c), block
    # a predictor chunk of 3 geometries splits pair 1 (replicas 2 and 3)
    _, ic, _, _, _ = _setup(name, n_saddles=3, chunk=3)
    d = _device(ic, R0, modes, 9, h, 0.0)
    assert np.array_equal(d['n_points'], a['n_points']) and np.array_equal(d['end'], a['end'])
    for k in ('R', 'E', 'fmax', 'R_path', 'E_path'):
        assert rel_err(np.nan_to_num(d[k]), np.nan_to_num(a[k])) < 1e-8, (k, rel_err(d[k], a[k]))


def test_pair_alone_and_among_many():
    import sgdml_b200

    gp, irc, R0, modes, h = _setup('n21_m6_s6', n_saddles=4)
    many = _device(irc, R0, modes, 8, h, 0.0)
    one = sgdml_b200.GDMLIRC(gp, _masses(gp.n_atoms), 1, E_to_eV=1.0, F_to_eV_Ang=1.0)
    assert np.array_equal(one.inv_mass, irc.inv_mass)
    alone = _device(one, R0[2:3], modes[2:3], 8, h, 0.0)
    for k in _KEYS:
        assert np.array_equal(alone[k], many[k][4:6], equal_nan=True), k


# ---------------------------------------------------------------------------------------------------- isolation, outputs
def test_isolated_from_predict_calls_and_other_handles():
    import torch

    import sgdml_b200

    gp, irc, R0, modes, h = _setup('n12_m8_s12')
    ref = _device(sgdml_b200.GDMLIRC(gp, _masses(gp.n_atoms), 2, E_to_eV=1.0, F_to_eV_Ang=1.0), R0,
                  modes, 8, h, 0.0)
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    rel._set_state_raw(np.repeat(R0, 2, axis=0)[:3])
    Rbig = np.tile(R0, (40, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((80, R0.shape[1]))
    E_before, F_before = gp.predict(Rbig)

    irc._set_state_raw(np.repeat(R0, 2, axis=0), step=7)
    gp.predict(Rbig)
    gp.predict_hvp(Rbig, np.ones_like(Rbig))
    rel._relax_raw('fire', 5, 0.0, 0.05, 0.1, 1.0)
    gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (80, 1, 1)))
    out = _device(irc, None, modes, 8, h, 0.0)
    assert _same(out, ref) and out['step'] == 7 and np.all(out['V'] == 0.0)
    E_after, F_after = gp.predict(Rbig)
    assert np.array_equal(E_before, E_after) and np.array_equal(F_before, F_after)


def test_host_device_and_null_outputs():
    """Host arrays, CUDA tensors and NULL for every output give the same final state and the same values."""
    import torch

    from sgdml_b200 import _lib

    gp, irc, R0, modes, h = _setup('n9_m16_s6')
    host = _device(irc, R0, modes, 9, h, 0.0)
    n, d = irc.n_replicas, R0.shape[1]
    outs = (torch.full((n, 9, d), 7.0, dtype=torch.float64, device='cuda'),
            torch.full((n, 9), 7.0, dtype=torch.float64, device='cuda'),
            torch.full((n,), 7, dtype=torch.int64, device='cuda'), torch.full((n,), 7, dtype=torch.int32, device='cuda'),
            torch.full((n,), 7.0, dtype=torch.float64, device='cuda'))
    irc._set_state_raw(np.repeat(R0, 2, axis=0))
    _lib.check(_lib.lib().sgdml_b200_irc_rk4(irc._handle, _lib.ptr(torch.from_numpy(modes).cuda()), 9, h, 0.0,
                                             *(_lib.ptr(x) for x in outs), _lib.current_stream()), 'irc_rk4')
    dev = dict(zip(('R_path', 'E_path', 'n_points', 'end', 'fmax'), (x.cpu().numpy() for x in outs)))
    st_dev = irc._get_state_raw()
    for k in dev:
        assert np.array_equal(dev[k], host[k], equal_nan=True), k
    irc._set_state_raw(np.repeat(R0, 2, axis=0))
    _lib.check(_lib.lib().sgdml_b200_irc_rk4(irc._handle, _lib.ptr(modes), 9, h, 0.0, None, None, None, None, None,
                                             _lib.current_stream()), 'irc_rk4')
    st_null = irc._get_state_raw()
    for st in (st_dev, st_null):
        for k, hk in (('R', 'R'), ('F', 'F'), ('E_pot', 'E'), ('V', 'V')):
            assert np.array_equal(st[k].cpu().numpy() if hasattr(st[k], 'cpu') else st[k], host[hk]), k


# ---------------------------------------------------------------------------------------------------- units and errors
def test_public_units():
    """GDMLIRC in eV / Angstrom / amu (a kcal/mol model, the default units) against its model-unit form, CUDA tensors
    in and out, broadcast saddles, and torch inputs that are not float64 CUDA tensors refused with the handle
    unchanged."""
    import math

    import torch

    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc
    from sgdml_b200.md import FS

    gp, _, R0, modes, _ = _setup('n9_m16_s6')
    N = gp.n_atoms
    m = np.linspace(1.0, 16.0, N)
    irc = sgdml_b200.GDMLIRC(gp, m, 2)
    pos, md = R0.reshape(2, N, 3), modes.reshape(2, N, 3)
    out = irc.run(pos, md, step=0.01, max_points=8, fmax=0.0, relax_ends=False)
    raw = sgdml_b200.GDMLIRC(gp, m, 2)
    raw._set_state_raw(np.repeat(R0, 2, axis=0))
    Rp, Ep, n, end, fm = raw._irc_raw(modes, 8, 0.01 / math.sqrt(kc * FS**2), 0.0)
    assert np.array_equal(out['positions'], Rp.reshape(2, 2, 8, N, 3), equal_nan=True)
    assert np.allclose(out['energies'], (Ep * kc).reshape(2, 2, 8), rtol=1e-15, equal_nan=True)
    assert np.array_equal(out['n_points'], n.reshape(2, 2)) and np.array_equal(out['end'], end.reshape(2, 2))
    assert np.allclose(out['fmax'], (fm * kc).reshape(2, 2), rtol=1e-15)
    k = np.arange(8)
    for b, sgn in ((0, 1.0), (1, -1.0)):
        nb = out['n_points'][0, b]
        assert np.allclose(out['s'][0, b, :nb], sgn * 0.01 * k[:nb], rtol=1e-15)
        assert np.all(np.isnan(out['s'][0, b, nb:]))
    t = irc.run(torch.from_numpy(pos).cuda(), torch.from_numpy(md).cuda(), step=0.01, max_points=8, fmax=0.0)
    assert t['positions'].is_cuda and t['s'].is_cuda and t['minima']['positions'].is_cuda and t['barriers'].is_cuda
    assert np.array_equal(t['positions'].cpu().numpy(), out['positions'], equal_nan=True)
    one = irc.run(pos[0], md[0], step=0.01, max_points=8, fmax=0.0, relax_ends=False)
    assert np.array_equal(one['positions'][1], one['positions'][0], equal_nan=True)
    before = irc._get_state_raw()
    m32 = torch.randn(2, N, 3, device='cuda')
    for kw in (dict(modes=m32), dict(modes=m32.long()), dict(modes=torch.from_numpy(md)),
               dict(saddles=torch.from_numpy(pos).cuda().float())):
        a = dict(saddles=pos, modes=md)
        a.update(kw)
        with pytest.raises(ValueError, match='float64 CUDA'):
            irc.run(a['saddles'], a['modes'], max_points=4)
        after = irc._get_state_raw()
        host = lambda x: x.cpu().numpy() if hasattr(x, 'cpu') else np.asarray(x)  # noqa: E731
        assert all(np.array_equal(host(before[k]), host(after[k])) for k in before)


def test_bad_input_and_handle_kinds_are_rejected():
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, irc, R0, modes, h = _setup('n9_m16_s6')
    L = _lib.lib()
    N3 = R0.shape[1]

    def call(H, m, n_rep=4, **kw):
        a = dict(mp=6, h=h, fmax=0.0)
        a.update(kw)
        out = (np.full((n_rep, 6, N3), 7.0), np.full((n_rep, 6), 7.0), np.full(n_rep, 7, dtype=np.int64),
               np.full(n_rep, 7, dtype=np.int32), np.full(n_rep, 7.0))
        rc = L.sgdml_b200_irc_rk4(H, None if m is None else m.ctypes.data, a['mp'], a['h'], a['fmax'],
                                  *(x.ctypes.data for x in out), _lib.current_stream())
        return rc, all(np.all(x == 7) for x in out)

    m = _masses(gp.n_atoms)
    fresh = sgdml_b200.GDMLIRC(gp, m, 2, E_to_eV=1.0, F_to_eV_Ang=1.0)
    assert call(fresh._handle, modes)[0] <= -1000  # no state
    irc._set_state_raw(np.repeat(R0, 2, axis=0), step=3)
    before = irc._get_state_raw()
    for bm in (np.stack([modes[0], np.full(N3, np.nan)]), np.stack([np.zeros(N3), modes[1]]),
               np.stack([modes[0], np.full(N3, np.inf)])):
        rc, untouched = call(irc._handle, np.ascontiguousarray(bm))
        assert rc <= -1000 and untouched
    for kw in (dict(mp=1), dict(mp=0), dict(mp=-3), dict(h=0.0), dict(h=-h), dict(h=np.nan), dict(h=np.inf),
               dict(fmax=-1.0), dict(fmax=np.nan)):
        rc, untouched = call(irc._handle, modes, **kw)
        assert rc <= -1000 and untouched, kw
    assert call(irc._handle, None)[0] <= -1000
    assert call(None, modes)[0] <= -1000
    after = irc._get_state_raw()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    # odd replica counts hold no pairs
    odd = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    odd._set_state_raw(np.repeat(R0, 2, axis=0)[:3])
    assert call(odd._handle, modes[:1], n_rep=3)[0] <= -1000

    # ring polymers, NPT, metadynamics and umbrella handles are refused, with state and outputs untouched
    model, Rq, _ = hvp_oracle.fixture_model('pbc_n6_m8')
    gpp = sgdml_b200.GDMLPredict(model)
    N = gpp.n_atoms
    d = 3 * N
    inv = np.ascontiguousarray(1.0 / np.linspace(1.0, 16.0, N))
    lat, linv = gpp.lat_and_inv
    L0 = np.ascontiguousarray(np.tile(lat.reshape(1, 9), (4, 1)))
    L0inv = np.ascontiguousarray(np.tile(linv.reshape(1, 9), (4, 1)))
    cv_type, cv_atoms = np.zeros(1, dtype=np.int32), np.array([[0, 1, 0, 0]], dtype=np.int64)
    cen, kap = np.ascontiguousarray([[1.0], [1.5]]), np.ascontiguousarray([[1.0], [1.0]])
    P = lambda x: x.ctypes.data  # noqa: E731
    Rs = np.ascontiguousarray(np.asarray(Rq, dtype=np.float64).reshape(-1, d)[np.arange(4) % len(Rq)])
    pm = np.random.default_rng(3).standard_normal((2, d))
    handles = []
    try:
        for create in (lambda H: L.sgdml_b200_pimd_create(H, gpp._handle, 2, 2, P(inv)),
                       lambda H: L.sgdml_b200_npt_create(H, gpp._handle, 4, P(inv), P(L0), P(L0inv)),
                       lambda H: L.sgdml_b200_metad_create(H, gpp._handle, 2, 2, P(inv), 1, P(cv_type), P(cv_atoms)),
                       lambda H: L.sgdml_b200_umbrella_create(H, gpp._handle, 2, 2, P(inv), 1, P(cv_type), P(cv_atoms),
                                                              P(cen), P(kap))):
            H = ctypes.c_void_p()
            _lib.check(create(ctypes.byref(H)), 'create')
            handles.append(H.value)
            _lib.check(L.sgdml_b200_md_set_state(H.value, P(Rs), None, 0, _lib.current_stream()), 'md_set_state')
            snap = [np.full((4, d), 1.5), np.full((4, d), 1.5), np.full((4, d), 1.5), np.full(4, 1.5)]
            _lib.check(L.sgdml_b200_md_get_state(H.value, *map(P, snap), None, _lib.current_stream()), 'get_state')
            out = (np.full((4, 6, d), 7.0), np.full((4, 6), 7.0), np.full(4, 7, dtype=np.int64),
                   np.full(4, 7, dtype=np.int32), np.full(4, 7.0))
            rc = L.sgdml_b200_irc_rk4(H.value, P(pm), 6, 1e-3, 0.0, *map(P, out), _lib.current_stream())
            assert rc <= -1000 and all(np.all(x == 7) for x in out)
            again = [np.full((4, d), 1.5), np.full((4, d), 1.5), np.full((4, d), 1.5), np.full(4, 1.5)]
            _lib.check(L.sgdml_b200_md_get_state(H.value, *map(P, again), None, _lib.current_stream()), 'get_state')
            assert all(np.array_equal(a, b) for a, b in zip(snap, again))
    finally:
        for H in handles:
            L.sgdml_b200_md_destroy(H)


# ---------------------------------------------------------------------------------------------------- physics
def test_irc_connects_the_double_well_saddle_to_both_minima():
    """On the model trained on the double-well hinge: relax A and B, CI-NEB to the saddle, one imaginary mode there;
    GDMLIRC follows it, with unequal masses and with all masses 12, down both branches (neither at max_points,
    energies strictly falling); after relax_ends one minimum matches A and the other B (Kabsch RMSD below 1e-3
    Angstrom, energies within 1e-7 eV), the forward branch being the one +mode points to (read off d01).  With equal
    masses the IRC is the Cartesian minimum-energy path: every interior CI-NEB image lies within 0.02 Angstrom of the
    IRC polyline.  The Vineyard rate from each minimum over the saddle is finite, and its barrier is the IRC's."""
    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc
    from sgdml_b200.md import kabsch_align
    from test_neb import _DW_PHI, _dw_hinge, _dw_task

    model = sgdml_b200.GDMLTrain().train(_dw_task())
    gp = sgdml_b200.GDMLPredict(model)
    dt, dtmax = 0.01 / np.sqrt(kc), 0.05 / np.sqrt(kc)
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=2)
    mins = rel.relax(_dw_hinge(_DW_PHI), fmax=1e-4 * kc, max_steps=3000, optimizer='fire', maxstep=0.05, dt=dt,
                     dtmax=dtmax)
    assert mins['converged'].all()
    A, B = mins['positions']
    E_A, E_B = mins['potential_energy']
    neb = sgdml_b200.GDMLNEB(gp, 9)
    band = neb.interpolate(A, B, align=True)
    k = 50.0 * kc
    neb.neb(band, fmax=0.05 * kc, max_steps=2000, k=k, climb=False, maxstep=0.05, dt=dt, dtmax=dtmax)
    ci = neb.neb(fmax=1e-6 * kc, max_steps=5000, k=k, climb=True, maxstep=0.05, dt=dt, dtmax=dtmax)
    assert ci['converged'].all()
    top = int(ci['climbing_image'][0])
    P = ci['positions'][0]
    saddle = P[top]

    d01 = lambda X: np.linalg.norm(X[0] - X[1])  # noqa: E731
    rmsd = lambda X, Y: np.sqrt(np.mean(np.sum((kabsch_align(X, Y) - Y) ** 2, -1)))  # noqa: E731
    for masses in (np.array([12.0, 16.0, 14.0, 1.0]), np.full(4, 12.0)):
        vib = sgdml_b200.GDMLVibrations(gp, masses)
        s = vib.analyse(saddle[None])
        assert s['n_imaginary'][0] == 1 and s['n_rigid'][0] == 6
        mode = s['modes'][0, 0]
        irc = sgdml_b200.GDMLIRC(gp, masses)
        out = irc.run(saddle, mode, step=0.02, max_points=2000, fmax=1e-4 * kc, relax_steps=3000)
        print('masses %s: points %s, end codes %s, barriers %s eV' % (masses.tolist(), out['n_points'].tolist(),
                                                                     out['end'].tolist(), out['barriers'].tolist()))
        assert np.all(out['end'] != 3) and np.all(out['n_points'] > 5)
        for b in range(2):
            n = out['n_points'][0, b]
            assert np.all(np.diff(out['energies'][0, b, :n]) < 0.0)
            assert np.all(np.isnan(out['energies'][0, b, n:]))
        assert out['minima']['converged'].all()
        fwd_to_B = d01(saddle + 1e-3 * mode / np.linalg.norm(mode)) > d01(saddle)
        want = (B, A) if fwd_to_B else (A, B)
        want_E = (E_B, E_A) if fwd_to_B else (E_A, E_B)
        for b in range(2):
            got = out['minima']['positions'][0, b]
            print('branch %d: RMSD %.3e A, dE %.3e eV' % (b, rmsd(got, want[b]),
                                                         out['minima']['potential_energy'][0, b] - want_E[b]))
            assert rmsd(got, want[b]) < 1e-3
            assert abs(out['minima']['potential_energy'][0, b] - want_E[b]) < 1e-7
        if masses[0] == masses[1]:
            # the IRC polyline, backward end to forward end through the saddle
            nf, nb = out['n_points'][0]
            line = np.concatenate([out['positions'][0, 1, :nb][::-1], out['positions'][0, 0, 1:nf]]).reshape(-1, 12)
            a, bb = line[:-1], line[1:]
            worst = 0.0
            for j in range(1, 8):
                x = P[j].ravel()
                t = np.clip(np.einsum('ij,ij->i', x - a, bb - a) / np.einsum('ij,ij->i', bb - a, bb - a), 0.0, 1.0)
                worst = max(worst, np.min(np.linalg.norm(a + t[:, None] * (bb - a) - x, axis=1)))
            print('largest distance of a CI-NEB image from the IRC: %.3e A' % worst)
            assert worst < 0.02
        for b in range(2):
            m = vib.analyse(out['minima']['positions'][0, b][None])
            r = sgdml_b200.harmonic_rate(m, s, 300.0)
            assert np.isfinite(r['rate'][0]) and r['rate'][0] > 0
            assert abs(r['barrier'][0] - out['barriers'][0, b]) < 1e-9
