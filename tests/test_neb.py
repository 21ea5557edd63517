"""The nudged elastic band on the device (sgdml_b200_neb_fire, sgdml_b200.GDMLNEB) against the NumPy restatement of
tests/neb_oracle.py driven by GDMLPredict.predict: every predictor form with and without a climbing image, int8 slices,
convergence counts and frozen bands, graph against plain launches, block lengths, chunks that split a band, a band
alone and among many, three-image bands, isolation from the predictor's own calls and from other handles, public
units and argument errors; and CI-NEB through the public interface on a double-well model trained in the test, whose
climbing image is checked to be a first-order saddle of the model with a Hessian from predict_hvp.
"""

import numpy as np
import pytest

import neb_oracle
import relax_oracle
from conftest import rel_err
from md_common import FIXTURES_MD, _cuda_forces

pytestmark = pytest.mark.gpu


def _setup(name, n_bands=2, P=5, chunk=0, slices=0):
    """(GDMLPredict, GDMLNEB in model units, R0 (n_bands P, 3N), scales {dt, maxstep, k}).  Band b runs linearly
    between two of the fixture's query geometries, its interior images displaced slightly off the line."""
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    model, Rq, _ = hvp_oracle.fixture_model(name)
    gp = sgdml_b200.GDMLPredict(model)
    if slices:
        gp.set_contraction_slices(slices)
    _lib.check(_lib.lib().sgdml_b200_set_predict_chunk(chunk), 'set_predict_chunk')
    try:
        neb = sgdml_b200.GDMLNEB(gp, P, n_bands=n_bands, E_to_eV=1.0, F_to_eV_Ang=1.0)
    finally:
        _lib.lib().sgdml_b200_set_predict_chunk(0)
    N = gp.n_atoms
    X = np.asarray(Rq, dtype=np.float64).reshape(-1, N, 3)
    a = X[np.arange(n_bands) % len(X)]
    b = X[(np.arange(n_bands) + 1) % len(X)]
    if len(X) == 1:
        b = b + 0.05 * np.random.default_rng(2).standard_normal(b.shape)
    band = neb.interpolate(a, b, P, align=False)
    band[:, 1:-1] += 2e-3 * np.random.default_rng(1).standard_normal(band[:, 1:-1].shape)
    R0 = band.reshape(n_bands * P, 3 * N)
    _, F0 = gp.predict(R0)
    f = float(np.max(np.abs(F0)))
    seg = float(np.max(np.abs(R0[1] - R0[0]))) + 1e-3
    return gp, neb, R0, {'dt': float(np.sqrt(0.01 / f)), 'maxstep': 0.05, 'k': 0.5 * f / seg}


def _device(neb, R0, steps, fmax, sc, climb):
    neb._set_state_raw(R0)
    n, c, fm, top = neb._neb_raw(steps, fmax, sc['k'], climb, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    st = neb._get_state_raw()
    return {'R': st['R'], 'F': st['F'], 'E': st['E_pot'], 'V': st['V'], 'step': st['step'], 'n_steps': n,
            'converged': c.astype(bool), 'fmax': fm, 'climbing': top}


def _oracle(gp, R0, P, steps, fmax, sc, climb):
    return neb_oracle.neb_fire(_cuda_forces(gp), R0, P, steps, fmax, sc['k'], climb, sc['maxstep'], sc['dt'],
                               10.0 * sc['dt'])


def _same(a, b, keys=('R', 'F', 'E', 'n_steps', 'converged', 'fmax', 'climbing')):
    return all(np.array_equal(a[k], b[k]) for k in keys)


def _check_against(dev, ref, R0, P, steps=None):
    assert rel_err(dev['R'], ref['R']) < 1e-12
    assert rel_err(dev['E'], ref['E']) < 1e-12
    assert rel_err(dev['fmax'], ref['fmax']) < 1e-12
    assert np.array_equal(dev['climbing'], ref['climbing'])
    ends = np.arange(len(R0)) % P
    ends = (ends == 0) | (ends == P - 1)
    assert np.array_equal(dev['R'][ends], R0[ends])  # the endpoints never move
    assert np.all(dev['V'] == 0.0) and dev['step'] == 0
    if steps is not None:
        assert np.all(dev['n_steps'] == steps) and not dev['converged'].any()


def _tie_free_fmax(gp, R0, P, steps, sc, climb):
    """A threshold between the bands' max |F_neb| after 2/3 of `steps`, at least 1e-6 (relative) from every value the
    convergence test compares with it; and the oracle's run at that threshold."""
    ref = _oracle(gp, R0, P, 2 * steps // 3, 0.0, sc, climb)
    f = np.sort(ref['fmax'])
    fmax = float(np.sqrt(f[len(f) // 2 - 1] * f[len(f) // 2]))
    for _ in range(50):
        out = _oracle(gp, R0, P, steps, fmax, sc, climb)
        if np.min(np.abs(out['tested'] / fmax - 1.0)) > 1e-6:
            return fmax, out
        fmax *= 1.0 + 1e-4
    raise AssertionError('no tie-free threshold')


# ---------------------------------------------------------------------------------------------------- against the oracle
@pytest.mark.parametrize('climb', [False, True])
@pytest.mark.parametrize('name', FIXTURES_MD)
def test_matches_restatement(name, climb):
    gp, neb, R0, sc = _setup(name)
    dev = _device(neb, R0, 12, 0.0, sc, climb)
    ref = _oracle(gp, R0, 5, 12, 0.0, sc, climb)
    print('%s climb=%s: R bit-identical to the restatement: %s, climbing %s' % (
        name, climb, np.array_equal(dev['R'], ref['R']), dev['climbing'].tolist()))
    _check_against(dev, ref, R0, 5, steps=12)
    assert rel_err(dev['R'], R0) > 1e-6  # it moved


@pytest.mark.parametrize('climb', [False, True])
def test_int8_slices(climb):
    gp, neb, R0, sc = _setup('big_n100_m2_s12', slices=6)
    dev = _device(neb, R0, 12, 0.0, sc, climb)
    ref = _oracle(gp, R0, 5, 12, 0.0, sc, climb)
    _check_against(dev, ref, R0, 5, steps=12)


@pytest.mark.parametrize('climb', [False, True])
def test_convergence_matches_restatement(climb):
    gp, neb, R0, sc = _setup('n9_m16_s6', n_bands=6)
    fmax, ref = _tie_free_fmax(gp, R0, 5, 40, sc, climb)
    dev = _device(neb, R0, 40, fmax, sc, climb)
    print('climb=%s: fmax %.6g, steps %s, converged %s' % (climb, fmax, dev['n_steps'].tolist(),
                                                          dev['converged'].tolist()))
    assert np.array_equal(dev['n_steps'], ref['n_steps'])
    assert np.array_equal(dev['converged'], ref['converged'])
    assert dev['converged'].any() and dev['n_steps'].min() < dev['n_steps'].max()
    _check_against(dev, ref, R0, 5)
    # converged bands are frozen: a second call takes no step and changes nothing
    neb._set_state_raw(dev['R'])
    before = neb._get_state_raw()
    n, c, fm, top = neb._neb_raw(10, fmax, sc['k'], climb, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    after = neb._get_state_raw()
    conv = dev['converged']
    assert np.all(n[conv] == 0) and np.all(c[conv] == 1)
    rows = np.repeat(conv, 5)
    assert np.array_equal(after['R'][rows], before['R'][rows])


# ---------------------------------------------------------------------------------------------------- bitwise equalities
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12', 'pbc_n6_m8'])
def test_graph_blocks_and_chunks(name, monkeypatch):
    from sgdml_b200 import _lib

    gp, neb, R0, sc = _setup(name, n_bands=3)
    fmax, _ = _tie_free_fmax(gp, R0, 5, 30, sc, True)
    a = _device(neb, R0, 30, fmax, sc, True)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _device(neb, R0, 30, fmax, sc, True)
    monkeypatch.delenv('SGDML_B200_GRAPH')
    assert _same(a, b)
    for block in (1, 7, 1000):
        _lib.check(_lib.lib().sgdml_b200_set_relax_block(block), 'set_relax_block')
        try:
            c = _device(neb, R0, 30, fmax, sc, True)
        finally:
            _lib.lib().sgdml_b200_set_relax_block(0)
        assert _same(a, c), block
    # a predictor chunk of 3 geometries splits every band of 5 images
    _, nc, _, _ = _setup(name, n_bands=3, chunk=3)
    d = _device(nc, R0, 30, fmax, sc, True)
    assert np.array_equal(d['n_steps'], a['n_steps']) and np.array_equal(d['converged'], a['converged'])
    for k in ('R', 'E', 'fmax'):
        assert rel_err(d[k], a[k]) < 1e-12, k


def test_band_alone_and_among_many():
    import sgdml_b200

    gp, neb, R0, sc = _setup('n21_m6_s6', n_bands=4)
    many = _device(neb, R0, 15, 0.0, sc, True)
    one = sgdml_b200.GDMLNEB(gp, 5, n_bands=1, E_to_eV=1.0, F_to_eV_Ang=1.0)
    alone = _device(one, R0[10:15], 15, 0.0, sc, True)
    assert np.array_equal(alone['R'], many['R'][10:15])
    assert np.array_equal(alone['E'], many['E'][10:15])
    assert alone['fmax'][0] == many['fmax'][2] and alone['climbing'][0] == many['climbing'][2]


def test_three_images(monkeypatch):
    gp, neb, R0, sc = _setup('n12_m8_s12', n_bands=4, P=3)
    a = _device(neb, R0, 15, 0.0, sc, True)
    ref = _oracle(gp, R0, 3, 15, 0.0, sc, True)
    _check_against(dev=a, ref=ref, R0=R0, P=3, steps=15)
    assert np.all(a['climbing'] == 1)
    monkeypatch.setenv('SGDML_B200_GRAPH', '0')
    b = _device(neb, R0, 15, 0.0, sc, True)
    assert _same(a, b)


# ---------------------------------------------------------------------------------------------------- isolation
def test_isolated_from_predict_calls_and_other_handles():
    import torch

    import sgdml_b200

    gp, neb, R0, sc = _setup('n12_m8_s12')
    ref = _device(sgdml_b200.GDMLNEB(gp, 5, n_bands=2, E_to_eV=1.0, F_to_eV_Ang=1.0), R0, 10, 0.0, sc, True)
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=3, E_to_eV=1.0, F_to_eV_Ang=1.0)
    rel._set_state_raw(R0[:3])
    Rbig = np.tile(R0, (9, 1)) + 1e-3 * np.random.default_rng(5).standard_normal((90, R0.shape[1]))
    E_before, F_before = gp.predict(Rbig)

    neb._set_state_raw(R0, step=7)
    gp.predict(Rbig)
    gp.predict_hvp(Rbig, np.ones_like(Rbig))
    rel._relax_raw('fire', 5, 0.0, 0.05, sc['dt'], 10.0 * sc['dt'])
    gp.predict_virial(torch.from_numpy(Rbig).cuda(), lattice=np.tile(20.0 * np.eye(3), (90, 1, 1)))
    n, c, fm, top = neb._neb_raw(10, 0.0, sc['k'], True, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    st = neb._get_state_raw()
    assert np.array_equal(st['R'], ref['R']) and np.array_equal(st['E_pot'], ref['E'])
    assert np.array_equal(fm, ref['fmax']) and np.array_equal(top, ref['climbing'])
    assert st['step'] == 7 and np.all(st['V'] == 0.0)
    E_after, F_after = gp.predict(Rbig)
    assert np.array_equal(E_before, E_after) and np.array_equal(F_before, F_after)

    # the same handle relaxes afterwards as relax_oracle does (every replica on its own)
    neb._set_state_raw(R0)
    neb._neb_raw(5, 0.0, sc['k'], True, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    neb._set_state_raw(R0)
    n, c, fm = neb._relax_raw('fire', 10, 0.0, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    want = relax_oracle.fire(_cuda_forces(gp), R0, 10, 0.0, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    assert rel_err(neb._get_state_raw()['R'], want['R']) < 1e-12
    assert rel_err(fm, want['fmax']) < 1e-12 and np.all(n == 10)


# ---------------------------------------------------------------------------------------------------- units and errors
def test_public_units():
    """GDMLNEB in eV / Angstrom (a kcal/mol model, the default units) against its model-unit form, and CUDA tensors in
    and out."""
    import torch

    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc

    gp, _, R0, sc = _setup('n9_m16_s6')
    N = gp.n_atoms
    neb = sgdml_b200.GDMLNEB(gp, 5, n_bands=2)
    images = R0.reshape(2, 5, N, 3)
    out = neb.neb(images, fmax=0.0, max_steps=10, k=0.3, climb=True, maxstep=0.1, dt=0.2, dtmax=0.8)
    raw = sgdml_b200.GDMLNEB(gp, 5, n_bands=2)
    raw._set_state_raw(R0)
    n, c, fm, top = raw._neb_raw(10, 0.0, 0.3 / kc, True, 0.1, 0.2 * np.sqrt(kc), 0.8 * np.sqrt(kc))
    st = raw._get_state_raw()
    assert np.array_equal(out['positions'], st['R'].reshape(2, 5, N, 3))
    assert np.allclose(out['energies'], st['E_pot'].reshape(2, 5) * kc, rtol=1e-15)
    assert np.allclose(out['forces'], st['F'].reshape(2, 5, N, 3) * kc, rtol=1e-15)
    assert np.allclose(out['fmax'], fm * kc, rtol=1e-15) and np.array_equal(out['n_steps'], n)
    assert np.array_equal(out['climbing_image'], top) and out['converged'].dtype == bool
    E = out['energies']
    assert np.array_equal(out['barrier'], E[:, 1:-1].max(1) - E[:, 0])
    t = neb.neb(torch.from_numpy(images).cuda(), fmax=0.0, max_steps=10, k=0.3, climb=True, maxstep=0.1, dt=0.2,
                dtmax=0.8)
    assert t['positions'].is_cuda and t['climbing_image'].is_cuda and t['barrier'].is_cuda
    assert np.array_equal(t['positions'].cpu().numpy(), out['positions'])
    assert np.array_equal(t['barrier'].cpu().numpy(), out['barrier'])
    # images=None continues from the current state
    again = neb.neb(fmax=0.0, max_steps=3, climb=True)
    assert not np.array_equal(again['positions'].cpu().numpy(), out['positions'])
    # one band may come without its band axis
    one = sgdml_b200.GDMLNEB(gp, 5)
    assert one.neb(images[0], fmax=0.0, max_steps=2)['positions'].shape == (1, 5, N, 3)
    with pytest.raises(ValueError):
        one.neb(images, fmax=0.0, max_steps=2)


def test_bad_input_is_rejected():
    import sgdml_b200
    from sgdml_b200 import _lib

    gp, neb, R0, sc = _setup('n9_m16_s6')
    L = _lib.lib()
    h = neb._handle
    fresh = sgdml_b200.GDMLNEB(gp, 5, n_bands=2, E_to_eV=1.0, F_to_eV_Ang=1.0)
    assert L.sgdml_b200_neb_fire(fresh._handle, 5, 10, 0.0, 0.1, 0, 0.1, 0.1, 1.0, None, None, None, None,
                                 None) <= -1000  # no state
    neb._set_state_raw(R0, step=3)
    neb._neb_raw(4, 0.0, sc['k'], True, sc['maxstep'], sc['dt'], 10.0 * sc['dt'])
    before = neb._get_state_raw()
    bad = [dict(n_images=2), dict(n_images=3), dict(n_images=4), dict(n_images=0), dict(n_images=-5),
           dict(max_steps=-1), dict(fmax=-1.0), dict(fmax=np.nan), dict(fmax=np.inf), dict(k=-0.1), dict(k=np.nan),
           dict(k=np.inf), dict(maxstep=0.0), dict(maxstep=np.nan), dict(dt=0.0), dict(dt=-1.0), dict(dt=np.inf),
           dict(dtmax=0.0), dict(dtmax=np.nan)]
    for kw in bad:
        a = dict(n_images=5, max_steps=10, fmax=0.0, k=0.1, maxstep=0.1, dt=0.1, dtmax=1.0)
        a.update(kw)
        out = (np.full(2, 7, dtype=np.int64), np.full(2, 7, dtype=np.int32), np.full(2, 7.0),
               np.full(2, 7, dtype=np.int32))
        rc = L.sgdml_b200_neb_fire(h, a['n_images'], a['max_steps'], a['fmax'], a['k'], 1, a['maxstep'], a['dt'],
                                   a['dtmax'], *(x.ctypes.data for x in out), _lib.current_stream())
        assert rc <= -1000, kw
        assert all(np.all(x == 7) for x in out)
    assert L.sgdml_b200_neb_fire(None, 5, 10, 0.0, 0.1, 0, 0.1, 0.1, 1.0, None, None, None, None, None) <= -1000
    # a ring-polymer handle holds no bands
    from md_common import md_fs_masses

    pimd = sgdml_b200.GDMLPathIntegralDynamics(gp, md_fs_masses(np.ones(gp.n_atoms)), 5, n_polymers=2, E_to_eV=1.0,
                                               F_to_eV_Ang=1.0)
    pimd._set_state_raw(R0)
    assert L.sgdml_b200_neb_fire(pimd._handle, 5, 10, 0.0, 0.1, 0, 0.1, 0.1, 1.0, None, None, None, None,
                                 None) <= -1000
    after = neb._get_state_raw()
    assert all(np.array_equal(before[k], after[k]) for k in before)
    with pytest.raises(ValueError):
        sgdml_b200.GDMLNEB(gp, 2)
    with pytest.raises(TypeError):
        neb.run(10, 0.5)


# ---------------------------------------------------------------------------------------------------- physics
# Four atoms: 2 and 3 on the z axis, 0 and 1 on the circle of radius _DW_RAD about it, held there by harmonic springs on
# every pair but (0, 1).  The hinge angle phi between atoms 0 and 1 is the one soft coordinate, and a double well in
# d01 = 2 _DW_RAD sin(phi / 2) puts minima at phi = 60 and 120 degrees with a barrier _DW_H between them at d01 = _DW_DC.
# The springs are stiff enough that the training geometries' wall energies lie well above the barrier, so a band has no
# way out of the sampled region that is downhill.
_DW_RAD, _DW_HALF, _DW_K, _DW_H = 1.2, 0.75, 10.0, 0.1
_DW_PHI = (np.pi / 3.0, 2.0 * np.pi / 3.0)
_DW_LO, _DW_HI = (2.0 * _DW_RAD * np.sin(p / 2.0) for p in _DW_PHI)
_DW_DC, _DW_W = 0.5 * (_DW_LO + _DW_HI), 0.5 * (_DW_HI - _DW_LO)


def _dw_hinge(phi):
    phi = np.atleast_1d(np.asarray(phi, dtype=np.float64))
    R = np.zeros((len(phi), 4, 3))
    R[:, 0] = [_DW_RAD, 0.0, 0.0]
    R[:, 1, 0] = _DW_RAD * np.cos(phi)
    R[:, 1, 1] = _DW_RAD * np.sin(phi)
    R[:, 2] = [0.0, 0.0, -_DW_HALF]
    R[:, 3] = [0.0, 0.0, _DW_HALF]
    return R


def _dw_pes(R):
    """(E, F) of the double-well hinge: springs 0.5 K (d - d_0)^2 on every pair but (0, 1), H (((d01 - dc)^2 - w^2) /
    w^2)^2 on d01."""
    r0 = _dw_hinge(_DW_PHI[0])[0]
    d0 = np.sqrt(((r0[:, None] - r0[None]) ** 2).sum(-1))
    R = np.asarray(R, dtype=np.float64).reshape(-1, 4, 3)
    diff = R[:, :, None] - R[:, None]
    d = np.sqrt((diff * diff).sum(-1)) + np.eye(4)
    mask = 1.0 - np.eye(4)
    mask[0, 1] = mask[1, 0] = 0.0
    ext = (d - d0 - np.eye(4)) * mask
    u = (d[:, 0, 1] - _DW_DC) ** 2 - _DW_W ** 2
    E = 0.25 * _DW_K * (ext * ext).sum((1, 2)) + _DW_H * u * u / _DW_W ** 4
    G = _DW_K * ext  # dE / d(d_ij)
    G[:, 0, 1] = G[:, 1, 0] = 4.0 * _DW_H * u * (d[:, 0, 1] - _DW_DC) / _DW_W ** 4
    return E, -(G[..., None] * diff / d[..., None]).sum(2)


def _dw_task():
    """Training geometries along the hinge (45 to 135 degrees) and along the straight line between the two wells, with
    0.05 Angstrom noise on every coordinate."""
    from sgdml_b200 import synth

    rng = np.random.default_rng(7)
    A, B = _dw_hinge(_DW_PHI)
    t = rng.uniform(-0.15, 1.15, 100)[:, None, None]
    R = np.concatenate([_dw_hinge(rng.uniform(np.pi / 4.0, 3.0 * np.pi / 4.0, 100)), A[None] + t * (B - A)[None]])
    R = R + 0.05 * rng.standard_normal(R.shape)
    task = synth.make_task(4, len(R), np.arange(4)[None], 2.0, seed=3)
    task['R_train'] = R
    task['E_train'], task['F_train'] = _dw_pes(R)
    task['dataset_theory'] = 'double_well_hinge'
    return task


def test_ci_neb_finds_a_first_order_saddle_of_a_trained_model():
    """Relax both minima of a model trained on the double-well hinge, run NEB and then CI-NEB between them through the
    public (eV, Angstrom) interface: the climbing image is a stationary point of the model with exactly one negative
    Hessian eigenvalue, the six rigid modes at zero, the highest energy on its band, and it sits on the barrier of the
    surface the model was trained on."""
    import sgdml_b200
    from sgdml_b200.intf.ase_calc import _KCAL_PER_MOL_IN_EV as kc

    model = sgdml_b200.GDMLTrain().train(_dw_task())
    gp = sgdml_b200.GDMLPredict(model)
    dt, dtmax = 0.01 / np.sqrt(kc), 0.05 / np.sqrt(kc)  # model units: 0.01 and 0.05
    rel = sgdml_b200.GDMLRelaxation(gp, n_replicas=2)
    mins = rel.relax(_dw_hinge(_DW_PHI), fmax=1e-4 * kc, max_steps=3000, optimizer='fire', maxstep=0.05, dt=dt,
                     dtmax=dtmax)
    assert mins['converged'].all(), mins['fmax']

    neb = sgdml_b200.GDMLNEB(gp, 9)
    band = neb.interpolate(mins['positions'][0], mins['positions'][1], align=True)
    k = 50.0 * kc  # eV / Angstrom^2: 50 in the model's kcal/mol / Angstrom^2
    plain = neb.neb(band, fmax=0.05 * kc, max_steps=2000, k=k, climb=False, maxstep=0.05, dt=dt, dtmax=dtmax)
    assert plain['converged'].all(), plain['fmax']
    fmax = 1e-6 * kc  # the rotational modes carry Hessian eigenvalues of order |F| |r| away from a stationary point
    ci = neb.neb(fmax=fmax, max_steps=5000, k=k, climb=True, maxstep=0.05, dt=dt, dtmax=dtmax)
    print('NEB %d steps, CI-NEB %d steps, energies %s eV' % (plain['n_steps'][0], ci['n_steps'][0], ci['energies'][0]))
    assert ci['converged'].all() and ci['fmax'][0] < fmax
    assert np.array_equal(ci['positions'][0, [0, -1]], band[[0, -1]])  # the endpoints never moved

    top = int(ci['climbing_image'][0])
    E = ci['energies'][0]
    assert 0 < top < 8 and E[top] == E.max()
    assert ci['barrier'][0] == E[top] - E[0]
    F = ci['forces'][0, top]
    assert np.sqrt((F * F).sum(-1)).max() < fmax  # the model's own force, not only its NEB projection

    # the model's Hessian at the climbing image, column by column from 3N Hessian-vector products (HV = -H V)
    x = ci['positions'][0, top].reshape(1, 12)
    H = np.empty((12, 12))
    for i in range(12):
        e = np.zeros((1, 12))
        e[0, i] = 1.0
        H[:, i] = -gp.predict_hvp(x, e)[0]
    assert np.max(np.abs(H - H.T)) < 1e-8 * np.max(np.abs(H))
    ev = np.linalg.eigvalsh(0.5 * (H + H.T))
    scale = np.max(np.abs(ev))
    print('Hessian eigenvalues at the climbing image: %s' % ev)
    assert (ev < -1e-6 * scale).sum() == 1
    assert np.sort(np.abs(ev))[5] < 1e-5 * scale  # translations and rotations
    assert np.sort(np.abs(ev))[6] > 1e-3 * scale  # and nothing else is soft

    # on the trained surface's barrier: d01 at the top of the double well, the barrier height within the fit
    X = x.reshape(4, 3)
    assert abs(np.linalg.norm(X[0] - X[1]) - _DW_DC) < 0.02
    assert abs(ci['barrier'][0] / kc - _DW_H) < 0.02
