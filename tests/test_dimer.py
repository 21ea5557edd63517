"""The dimer search on the device (sgdml_b200_dimer_fire, sgdml_b200.GDMLDimer) against the NumPy restatement of
tests/dimer_oracle.py driven by GDMLPredict.predict: every predictor form, int8 slices, rotating and translating-only
dimers, graph against plain launches, block lengths, chunks that split a dimer's pair, a dimer alone and among many,
isolation from the predictor's own calls and from other handles, public units and argument errors; and searches
through the public interface on the double-well hinge model of tests/test_neb.py, trained in the test, whose end
points are checked to be its first-order saddle with a Hessian from predict_hvp and against a CI-NEB climbing image.
"""

import numpy as np
import pytest

import dimer_oracle
from conftest import rel_err
from md_common import FIXTURES_MD, _cuda_forces
from test_neb import _DW_DC, _DW_PHI, _dw_hinge, _dw_task

pytestmark = pytest.mark.gpu

_CT, _ST = np.cos(np.pi / 4), np.sin(np.pi / 4)
_KEYS = ('R', 'F', 'E', 'modes', 'curvature', 'n_steps', 'n_rot', 'converged', 'fmax')


def _setup(name, n_dimers=2, chunk=0, slices=0):
    """(GDMLPredict, GDMLDimer in model units, R0 (2 n_dimers, 3N), modes (n_dimers, 3N), scales).  The centres are
    the fixture's query geometries, the modes seeded normals."""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    gp = sgdml_b200.GDMLPredict(model)
    if slices:
        gp.set_contraction_slices(slices)
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        dim = sgdml_b200.GDMLDimer(gp, n_dimers, E_to_eV=1.0, F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    N = gp.n_atoms
    X = np.asarray(Rq, dtype=np.float64).reshape(-1, 3 * N)
    R0 = np.repeat(X[np.arange(n_dimers) % len(X)], 2, axis=0)
    R0[::2] += 1e-2 * np.random.default_rng(1).standard_normal(R0[::2].shape)
    modes = np.random.default_rng(2).standard_normal((n_dimers, 3 * N))
    _, F0 = gp.predict(R0)
    f = float(np.max(np.abs(F0)))
    return gp, dim, R0, modes, {'dt': float(np.sqrt(0.01 / f)), 'maxstep': 0.05, 'D': 1e-3, 'rot_min': 0.0}


def _args(sc, steps, fmax):
    return (steps, fmax, sc['D'], _CT, _ST, sc['rot_min'], sc['maxstep'], sc['dt'], 10.0 * sc['dt'])


def _device(dim, R0, modes, steps, fmax, sc):
    if R0 is not None:
        dim._set_state_raw(R0)
    n, c, fm, cu, nr, md = dim._dimer_raw(modes, *_args(sc, steps, fmax))
    st = dim._get_state_raw()
    return {'R': st['R'], 'F': st['F'], 'E': st['E_pot'], 'V': st['V'], 'step': st['step'], 'n_steps': n,
            'converged': c.astype(bool), 'fmax': fm, 'curvature': cu, 'n_rot': nr, 'modes': md}


def _oracle(gp, R0, modes, steps, fmax, sc):
    project = 'translations' if gp.lat_and_inv is not None else 'rigid'
    return dimer_oracle.search(_cuda_forces(gp), R0, modes, *_args(sc, steps, fmax), project_=project)


def _same(a, b, keys=_KEYS):
    return all(np.array_equal(a[k], b[k]) for k in keys)


def _check_against(dev, ref):
    bad = [k for k in _KEYS if not np.array_equal(dev[k], ref[k])]
    assert not bad, (bad, [rel_err(dev[k], ref[k]) for k in bad])
    assert np.all(dev['V'] == 0.0) and dev['step'] == 0


# ---------------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_matches_restatement(name):
    gp, dim, R0, modes, sc = _setup(name)
    dev = _device(dim, R0, modes, 12, 0.0, sc)
    ref = _oracle(gp, R0, modes, 12, 0.0, sc)
    print('%s: rotations %s, translations %s, curvatures %s' % (name, dev['n_rot'].tolist(), dev['n_steps'].tolist(),
                                                                dev['curvature'].tolist()))
    _check_against(dev, ref)
    assert np.all(dev['n_rot'] == 6) and np.all(dev['n_steps'] == 6)  # every iteration rotates once
    assert rel_err(dev['R'][::2], R0[::2]) > 1e-6  # the centres moved


@pytest.mark.parametrize('rot_min', [1e30, 'mid'])
def test_translation_only_and_mixed(rot_min):
    """rot_min above every rotational force: no rotation, one translation per force evaluation; in the middle of them:
    both kinds of iteration in one call."""
    gp, dim, R0, modes, sc = _setup('n12_m8_s12', n_dimers=4)
    if rot_min == 'mid':  # between the second and third of the four rotational forces at the start
        R = R0.copy()
        N = [dimer_oracle.init_mode(modes[d], R0[2 * d]) for d in range(4)]
        for d in range(4):
            R[2 * d + 1] = R0[2 * d] + sc['D'] * N[d]
        _, F = _cuda_forces(gp)(R)
        f = []
        for d in range(4):
            G = (F[2 * d + 1] - F[2 * d]) / sc['D']
            P = G - dimer_oracle.block_sum(G * N[d]) * N[d]
            f.append(np.sqrt(dimer_oracle.block_sum(P * P)))
        f = np.sort(f)
        sc['rot_min'] = float(np.sqrt(f[1] * f[2]))
    else:
        sc['rot_min'] = rot_min
    dev = _device(dim, R0, modes, 14, 0.0, sc)
    ref = _oracle(gp, R0, modes, 14, 0.0, sc)
    print('rot_min %g: rotations %s, translations %s' % (sc['rot_min'], dev['n_rot'].tolist(), dev['n_steps'].tolist()))
    _check_against(dev, ref)
    if rot_min == 'mid':
        assert dev['n_rot'].max() > 0 and dev['n_rot'].min() < dev['n_rot'].max()
    else:
        assert np.all(dev['n_rot'] == 0) and np.all(dev['n_steps'] == 14)


def test_int8_slices():
    gp, dim, R0, modes, sc = _setup('big_n100_m2_s12', slices=6)
    _check_against(_device(dim, R0, modes, 12, 0.0, sc), _oracle(gp, R0, modes, 12, 0.0, sc))


def test_convergence_matches_restatement():
    """A threshold between the dimers' max |F0| late in the run: the counts, the frozen dimers and every output as the
    restatement's; a second call on converged dimers takes no step."""
    gp, dim, R0, modes, sc = _setup('n9_m16_s6', n_dimers=6)
    probe = _oracle(gp, R0, modes, 30, 0.0, sc)
    neg = np.sort(probe['fmax'][probe['curvature'] < 0.0])
    fmax = float(neg[len(neg) // 2]) * 1.5 if len(neg) else float(np.median(probe['fmax']))
    dev = _device(dim, R0, modes, 40, fmax, sc)
    ref = _oracle(gp, R0, modes, 40, fmax, sc)
    print('fmax %.6g: steps %s, rotations %s, converged %s, curvatures %s' % (
        fmax, dev['n_steps'].tolist(), dev['n_rot'].tolist(), dev['converged'].tolist(), dev['curvature'].tolist()))
    _check_against(dev, ref)
    assert np.all(dev['curvature'][dev['converged']] < 0.0)
    if dev['converged'].any():
        again = _device(dim, None, None, 10, fmax, sc)
        conv = dev['converged']
        assert np.all(again['n_steps'][conv] == 0) and np.all(again['converged'][conv])
        assert np.array_equal(again['R'][np.repeat(conv, 2)][::2], dev['R'][np.repeat(conv, 2)][::2])


# ---------------------------------------------------------------------------------------------------- bitwise equalities
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12', 'pbc_n6_m8'])
def test_graph_blocks_and_chunks(name, monkeypatch):
    from sgdml_b200 import _lib

    gp, dim, R0, modes, sc = _setup(name, n_dimers=3)
    a = _device(dim, R0, modes, 30, 0.0, sc)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _device(dim, R0, modes, 30, 0.0, sc)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    for block in (1, 7, 1000):
        _lib.check(_lib.lib().sgdml_b200_set_relax_block(block), 'set_relax_block')
        try:
            c = _device(dim, R0, modes, 30, 0.0, sc)
        finally:
            _lib.lib().sgdml_b200_set_relax_block(0)
        assert _same(a, c), block
    # a predictor chunk of 3 geometries splits the pair of dimer 1
    _, dc, _, _, _ = _setup(name, n_dimers=3, chunk=3)
    d = _device(dc, R0, modes, 30, 0.0, sc)
    assert np.array_equal(d['n_steps'], a['n_steps']) and np.array_equal(d['n_rot'], a['n_rot'])
    for k in ('R', 'E', 'fmax', 'modes', 'curvature'):
        assert rel_err(d[k], a[k]) < 1e-8, (k, rel_err(d[k], a[k]))


def test_dimer_alone_and_among_many():
    import sgdml_b200

    gp, dim, R0, modes, sc = _setup('n21_m6_s6', n_dimers=4)
    many = _device(dim, R0, modes, 15, 0.0, sc)
    one = sgdml_b200.GDMLDimer(gp, 1, E_to_eV=1.0, F_to_eV_Ang=1.0)
    alone = _device(one, R0[4:6], modes[2:3], 15, 0.0, sc)
    for k in ('R', 'F', 'E'):
        assert np.array_equal(alone[k], many[k][4:6]), k
    for k in ('modes', 'curvature', 'n_rot', 'n_steps', 'fmax'):
        assert np.array_equal(alone[k][0], many[k][2]), k


# ---------------------------------------------------------------------------------------------------- isolation
def test_isolated_from_predict_calls_and_other_handles():
    import torch

    import sgdml_b200

    gp, dim, R0, modes, sc = _setup('n12_m8_s12')
    ref = _device(sgdml_b200.GDMLDimer(gp, 2, E_to_eV=1.0, F_to_eV_Ang=1.0), R0, modes, 10, 0.0, sc)
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    rel._set_state_raw(R0[:3])
    Rbig = np.tile(R0, (20, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((80, R0.shape[1]))
    E_before, F_before = gp.predict(Rbig)

    dim._set_state_raw(R0, step=7)
    gp.predict(Rbig)
    gp.predict_hvp(Rbig, np.ones_like(Rbig))
    rel._relax_raw('fire', 5, 0.0, 0.05, sc['dt'], 10.0 * sc['dt'])
    gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (80, 1, 1)))
    out = _device(dim, None, modes, 10, 0.0, sc)
    assert _same(out, ref) and out['step'] == 7 and np.all(out['V'] == 0.0)
    E_after, F_after = gp.predict(Rbig)
    assert np.array_equal(E_before, E_after) and np.array_equal(F_before, F_after)
    # the same handle relaxes afterwards as relax_oracle does (every replica on its own)
    import relax_oracle

    dim._set_state_raw(R0)
    n, c, fm = dim._relax_raw('fire', 10, 0.0, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    want = relax_oracle.fire(_cuda_forces(gp), R0, 10, 0.0, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    assert rel_err(dim._get_state_raw()['R'], want['R']) < 1e-12 and np.all(n == 10)


def test_modes_are_kept_between_calls():
    """modes = NULL continues with the handle's modes: two calls of 6 and 6 force evaluations against the restatement
    started again from the first call's centres and modes."""
    gp, dim, R0, modes, sc = _setup('n9_m16_s6')
    first = _device(dim, R0, modes, 6, 0.0, sc)
    second = _device(dim, None, None, 6, 0.0, sc)
    ref = _oracle(gp, first['R'], first['modes'], 6, 0.0, sc)
    _check_against(second, ref)


# ---------------------------------------------------------------------------------------------------- units and errors
def test_public_units():
    """GDMLDimer in eV / Angstrom (a kcal/mol model, the default units) against its model-unit form, CUDA tensors in
    and out, broadcast positions and the seeded default modes."""
    import math

    import torch

    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc

    gp, _, R0, modes, sc = _setup('n9_m16_s6')
    N = gp.n_atoms
    dim = sgdml_b200.GDMLDimer(gp, 2)
    pos = R0[::2].reshape(2, N, 3)
    kw = dict(fmax=0.0, max_steps=10, separation=2e-3, trial_angle=0.5, rot_min=0.05, maxstep=0.1, dt=0.2, dtmax=0.8)
    out = dim.search(pos, modes.reshape(2, N, 3), **kw)
    raw = sgdml_b200.GDMLDimer(gp, 2)
    raw._set_state_raw(np.repeat(R0[::2], 2, axis=0))
    n, c, fm, cu, nr, md = raw._dimer_raw(modes, 10, 0.0, 2e-3, math.cos(0.5), math.sin(0.5), 0.05 / kc, 0.1,
                                          0.2 * np.sqrt(kc), 0.8 * np.sqrt(kc))
    st = raw._get_state_raw()
    assert np.array_equal(out['positions'], st['R'][::2].reshape(2, N, 3))
    assert np.array_equal(out['mode'], md.reshape(2, N, 3))
    assert np.allclose(out['potential_energy'], st['E_pot'][::2] * kc, rtol=1e-15)
    assert np.allclose(out['forces'], st['F'][::2].reshape(2, N, 3) * kc, rtol=1e-15)
    assert np.allclose(out['curvature'], cu * kc, rtol=1e-15) and np.allclose(out['fmax'], fm * kc, rtol=1e-15)
    assert np.array_equal(out['n_steps'], n) and np.array_equal(out['n_rotations'], nr)
    assert out['converged'].dtype == bool
    t = dim.search(torch.from_numpy(pos).cuda(), torch.from_numpy(modes.reshape(2, N, 3)).cuda(), **kw)
    assert t['positions'].is_cuda and t['mode'].is_cuda and t['curvature'].is_cuda
    assert np.array_equal(t['positions'].cpu().numpy(), out['positions'])
    # positions=None continues; modes=None keeps the modes
    again = dim.search(fmax=0.0, max_steps=3)
    assert not np.array_equal(again['positions'].cpu().numpy(), out['positions'])
    # (N, 3) is copied to every dimer; the first call's default modes are seeded normals
    a = sgdml_b200.GDMLDimer(gp, 2).search(pos[0], fmax=0.0, max_steps=4, seed=3)
    b = sgdml_b200.GDMLDimer(gp, 2).search(np.stack([pos[0], pos[0]]),
                                           np.random.default_rng(3).standard_normal((2, N, 3)), fmax=0.0, max_steps=4)
    assert np.array_equal(a['positions'], b['positions']) and np.array_equal(a['mode'], b['mode'])
    with pytest.raises(ValueError):
        dim.search(pos[:, :2], fmax=0.0, max_steps=2)
    # torch modes or positions that are not float64 CUDA tensors are refused with the handle unchanged
    before = dim._get_state_raw()
    m32 = torch.randn(2, N, 3, device='cuda')
    for kw in (dict(modes=m32), dict(positions=pos, modes=m32), dict(modes=m32.long()),
               dict(modes=torch.from_numpy(modes.reshape(2, N, 3))),
               dict(positions=torch.from_numpy(pos).cuda().float())):
        with pytest.raises(ValueError, match='float64 CUDA'):
            dim.search(fmax=0.0, max_steps=2, **kw)
        after = dim._get_state_raw()
        host = lambda x: x.cpu().numpy() if hasattr(x, 'cpu') else np.asarray(x)  # noqa: E731
        assert all(np.array_equal(host(before[k]), host(after[k])) for k in before)


def test_bad_input_is_rejected():
    import sgdml_b200
    from md_common import md_fs_masses
    from sgdml_b200 import _lib

    gp, dim, R0, modes, sc = _setup('n9_m16_s6')
    L = _lib.lib()
    N3 = R0.shape[1]

    def call(h, m, **kw):
        a = dict(max_steps=10, fmax=0.0, D=1e-3, ct=_CT, st=_ST, rot_min=0.0, maxstep=0.1, dt=0.1, dtmax=1.0)
        a.update(kw)
        out = (np.full(2, 7, dtype=np.int64), np.full(2, 7, dtype=np.int32), np.full(2, 7.0), np.full(2, 7.0),
               np.full(2, 7, dtype=np.int64), np.full((2, N3), 7.0))
        rc = L.sgdml_b200_dimer_fire(h, None if m is None else m.ctypes.data, a['max_steps'], a['fmax'], a['D'],
                                     a['ct'], a['st'], a['rot_min'], a['maxstep'], a['dt'], a['dtmax'],
                                     *(x.ctypes.data for x in out), _lib.current_stream())
        return rc, all(np.all(x == 7) for x in out)

    fresh = sgdml_b200.GDMLDimer(gp, 2, E_to_eV=1.0, F_to_eV_Ang=1.0)
    assert call(fresh._handle, modes)[0] <= -1000  # no state
    fresh._set_state_raw(R0)
    assert call(fresh._handle, None)[0] <= -1000  # no modes yet
    dim._set_state_raw(R0, step=3)
    twin = sgdml_b200.GDMLDimer(gp, 2, E_to_eV=1.0, F_to_eV_Ang=1.0)
    twin._set_state_raw(R0, step=3)
    for h in (dim, twin):
        h._dimer_raw(modes, *_args(sc, 4, 0.0))
    before = dim._get_state_raw()
    c1 = before['R'][2].reshape(-1, 3)  # dimer 1's centre now
    rot = np.cross(np.array([0.0, 0.0, 1.0]), c1 - c1.mean(0)).ravel()
    bad_modes = [np.stack([modes[0], rot]), np.stack([modes[0], np.full(N3, np.nan)]), np.zeros((2, N3)),
                 np.stack([np.tile([1.0, -2.0, 0.5], N3 // 3), modes[1]])]
    for m in bad_modes:
        rc, untouched = call(dim._handle, np.ascontiguousarray(m))
        assert rc <= -1000 and untouched
    bad = [dict(max_steps=-1), dict(fmax=-1.0), dict(fmax=np.nan), dict(D=0.0), dict(D=-1e-3), dict(D=np.inf),
           dict(ct=0.0), dict(st=-_ST), dict(ct=0.6, st=0.6), dict(ct=np.nan), dict(rot_min=-0.1),
           dict(rot_min=np.nan), dict(maxstep=0.0), dict(dt=0.0), dict(dt=np.inf), dict(dtmax=-1.0)]
    for kw in bad:
        rc, untouched = call(dim._handle, modes, **kw)
        assert rc <= -1000 and untouched, kw
    assert call(None, modes)[0] <= -1000
    # odd replica counts, ring polymers and metadynamics handles hold no dimers
    odd = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    odd._set_state_raw(R0[:3])
    assert call(odd._handle, modes[:1])[0] <= -1000
    pimd = sgdml_b200.GDMLPathIntegralDynamics(gp, md_fs_masses(np.ones(gp.n_atoms)), 2, n_polymers=2, E_to_eV=1.0,
                                               F_to_eV_Ang=1.0)
    pimd._set_state_raw(R0)
    assert call(pimd._handle, modes)[0] <= -1000
    metad = sgdml_b200.GDMLMetadynamics(gp, md_fs_masses(np.ones(gp.n_atoms)), [('distance', (0, 1))], n_walkers=4,
                                        E_to_eV=1.0, F_to_eV_Ang=1.0)
    metad._set_state_raw(R0)
    assert call(metad._handle, modes)[0] <= -1000
    after = dim._get_state_raw()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    # the kept modes are untouched too: a continuation equals the twin's, which saw no rejected call
    a = _device(dim, None, None, 5, 0.0, sc)
    b = _device(twin, None, None, 5, 0.0, sc)
    assert _same(a, b)
    with pytest.raises(TypeError):
        dim.run(10, 0.5)


# ---------------------------------------------------------------------------------------------------- physics
def test_dimers_find_the_double_well_saddle_of_a_trained_model():
    """Eight dimers started 12 degrees along the hinge from minimum A of the model trained on the double-well hinge
    (0.02 Angstrom of seeded noise), with modes along the aligned A -> B difference plus seeded noise, all end on the
    model's first-order saddle: one negative Hessian eigenvalue (from predict_hvp) with the six rigid modes at zero, the
    mode along its eigenvector and the curvature its eigenvalue, d01 at the top of the double well, and the energy of
    a CI-NEB climbing image computed here."""
    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc
    from sgdml_b200.md import kabsch_align

    model = sgdml_b200.GDMLTrain().train(_dw_task())
    gp = sgdml_b200.GDMLPredict(model)
    dt, dtmax = 0.01 / np.sqrt(kc), 0.05 / np.sqrt(kc)  # model units: 0.01 and 0.05
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=2)
    mins = rel.relax(_dw_hinge(_DW_PHI), fmax=1e-4 * kc, max_steps=3000, optimizer='fire', maxstep=0.05, dt=dt,
                     dtmax=dtmax)
    assert mins['converged'].all(), mins['fmax']
    A, B = mins['positions']

    neb = sgdml_b200.GDMLNEB(gp, 9)
    band = neb.interpolate(A, B, align=True)
    k = 50.0 * kc
    neb.neb(band, fmax=0.05 * kc, max_steps=2000, k=k, climb=False, maxstep=0.05, dt=dt, dtmax=dtmax)
    ci = neb.neb(fmax=1e-6 * kc, max_steps=5000, k=k, climb=True, maxstep=0.05, dt=dt, dtmax=dtmax)
    assert ci['converged'].all()
    E_ci = ci['energies'][0, int(ci['climbing_image'][0])]

    # From A itself the 0.02 Angstrom of noise decides which way along the hinge a dimer climbs, and the way towards
    # smaller angles leaves the sampled region (on the surface the model was trained on, it ends on a saddle of the
    # springs at d01 = 0.95).  So the start moves 12 degrees along the hinge, atom 1 turned about the z axis.
    n = 8
    rng = np.random.default_rng(21)
    t = np.deg2rad(12.0)
    turn = np.array([[np.cos(t), -np.sin(t), 0.0], [np.sin(t), np.cos(t), 0.0], [0.0, 0.0, 1.0]])
    base = A.copy()
    base[1] = turn @ A[1]
    start = base[None] + 0.02 * rng.standard_normal((n, 4, 3))
    diff = kabsch_align(B, A) - A
    modes = diff[None] + 0.1 * np.linalg.norm(diff) * rng.standard_normal((n, 4, 3))
    fmax = 1e-6 * kc
    dim = sgdml_b200.GDMLDimer(gp, n)
    out = dim.search(start, modes, fmax=fmax, max_steps=20000, rot_min=1e-3 * kc, maxstep=0.05, dt=dt, dtmax=dtmax)
    print('dimer: translations %s, rotations %s, curvatures %s eV/A^2' % (
        out['n_steps'].tolist(), out['n_rotations'].tolist(), out['curvature'].tolist()))
    assert out['converged'].all(), (out['fmax'], out['n_steps'])
    assert np.all(out['fmax'] < fmax)
    for d in range(n):
        x = out['positions'][d].reshape(1, 12)
        H = np.empty((12, 12))
        for i in range(12):
            e = np.zeros((1, 12))
            e[0, i] = 1.0
            H[:, i] = -gp.predict_hvp(x, e)[0]
        ev, vec = np.linalg.eigh(0.5 * (H + H.T))
        scale = np.max(np.abs(ev))
        assert (ev < -1e-6 * scale).sum() == 1, ev
        assert np.sort(np.abs(ev))[5] < 1e-5 * scale  # translations and rotations
        assert abs(out['mode'][d].ravel() @ vec[:, 0]) > 0.99
        assert abs(out['curvature'][d] / kc / ev[0] - 1.0) < 1e-3, (out['curvature'][d] / kc, ev[0])
        X = x.reshape(4, 3)
        assert abs(np.linalg.norm(X[0] - X[1]) - _DW_DC) < 0.02
        assert abs(out['potential_energy'][d] / E_ci - 1.0) < 1e-6, (out['potential_energy'][d], E_ci)
