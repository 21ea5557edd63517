"""Which entry points take which kind of dynamics handle: every sgdml_b200_md_*, _remd_*, _pimd_*, _relax_*, _neb_*,
_dimer_*, _npt_* and _metad_* entry point on a handle of every kind, against the table next to sgdml_b200_md_create in
include/sgdml_b200.h.

GPU: five handles of n_rep = 6 replicas of the periodic pbc_n6_m8 model (plain from sgdml_b200_md_create and from
sgdml_b200_pimd_create with one bead, a ring polymer of two beads, NPT and metadynamics), each with a state.  Every
entry point is called on every handle with arguments valid for that entry point and a few steps.  An accepted call
succeeds; a refused one returns an argument error, writes none of its outputs and changes neither the handle's state
nor, where the kind has them, its cells or hills.
"""

import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_REP = 6
PLAIN, RING, NPT, METAD = 'plain', 'ring', 'npt', 'metad'
ACCEPTS = {
    'md_set_state': {PLAIN, RING, NPT, METAD},
    'md_get_state': {PLAIN, RING, NPT, METAD},
    'md_run': {PLAIN},
    'remd_run': {PLAIN},
    'neb_fire': {PLAIN},
    'dimer_fire': {PLAIN},
    'pimd_run': {PLAIN, RING},
    'relax_fire': {PLAIN, RING},
    'relax_lbfgs': {PLAIN, RING},
    'npt_run': {NPT},
    'npt_set_cells': {NPT},
    'npt_get_cells': {NPT},
    'metad_run': {METAD},
    'metad_get_hills': {METAD},
    'metad_set_hills': {METAD},
    'metad_get_bias': {METAD},
}


def _full(shape, dtype=np.float64):
    """an output filled with a sentinel no call writes"""
    return np.full(shape, np.iinfo(dtype).max if np.issubdtype(dtype, np.integer) else 1.5, dtype=dtype)


def _p(x):
    return None if x is None else x.ctypes.data


def test_every_entry_point_on_every_kind():
    import hvp_oracle
    import sgdml_b200
    from sgdml_b200 import _lib

    L = _lib.lib()
    st = _lib.current_stream()
    model, Rq, _ = hvp_oracle.fixture_model('pbc_n6_m8')
    gp = sgdml_b200.GDMLPredict(model)
    N = gp.n_atoms
    d = 3 * N
    inv_mass = 1.0 / np.linspace(1.0, 16.0, N)
    s = inv_mass.repeat(3)
    Rc = np.asarray(Rq, dtype=np.float64).reshape(Rq.shape[0], -1)
    R0 = np.ascontiguousarray(Rc[np.arange(N_REP) % Rc.shape[0]])
    _, F0 = gp.predict(R0[:1])
    dt = float(np.sqrt(2e-3 / max(np.max(np.abs(F0 * s)), 1e-300)))
    V0 = np.random.default_rng(2).standard_normal(R0.shape) * 1e-3 / dt
    kT, gamma = float(np.mean(V0 * V0 / s)), 0.1 / dt
    lat, inv = gp.lat_and_inv
    L0 = np.ascontiguousarray(np.tile(lat.reshape(1, 9), (N_REP, 1)))
    L0inv = np.ascontiguousarray(np.tile(inv.reshape(1, 9), (N_REP, 1)))
    n_groups = 3
    cv_type, cv_atoms = np.zeros(1, dtype=np.int32), np.array([[0, 1, 0, 0]], dtype=np.int64)

    handles = {}
    try:
        for name, create in (
                ('plain', lambda h: L.sgdml_b200_md_create(h, gp._handle, N_REP, _p(inv_mass))),
                ('plain1', lambda h: L.sgdml_b200_pimd_create(h, gp._handle, N_REP, 1, _p(inv_mass))),
                ('ring', lambda h: L.sgdml_b200_pimd_create(h, gp._handle, N_REP // 2, 2, _p(inv_mass))),
                ('npt', lambda h: L.sgdml_b200_npt_create(h, gp._handle, N_REP, _p(inv_mass), _p(L0), _p(L0inv))),
                ('metad', lambda h: L.sgdml_b200_metad_create(h, gp._handle, n_groups, N_REP // n_groups, _p(inv_mass),
                                                              1, _p(cv_type), _p(cv_atoms)))):
            h = ctypes.c_void_p()
            _lib.check(create(ctypes.byref(h)), name)
            handles[name] = h.value
        kinds = {'plain': PLAIN, 'plain1': PLAIN, 'ring': RING, 'npt': NPT, 'metad': METAD}

        def snapshot(H, kind):
            """the handle's state, and its cells or hills where its kind has them"""
            out = [_full((N_REP, d)), _full((N_REP, d)), _full((N_REP, d)), _full(N_REP), _full(1, np.uint64)]
            _lib.check(L.sgdml_b200_md_get_state(H, *map(_p, out), st), 'md_get_state')
            if kind == NPT:
                cells = [_full((N_REP, 9)) for _ in range(3)]
                _lib.check(L.sgdml_b200_npt_get_cells(H, *map(_p, cells), st), 'npt_get_cells')
                out += cells
            if kind == METAD:
                n = _full(n_groups, np.int64)
                _lib.check(L.sgdml_b200_metad_get_hills(H, _p(n), None, None, None, st), 'metad_get_hills')
                t = int(n.sum())
                hills = [_full((t, 1)), _full((t, 1)), _full(t)]
                _lib.check(L.sgdml_b200_metad_get_hills(H, _p(n), *map(_p, hills), st), 'metad_get_hills')
                bias = [_full((N_REP, 1)), _full(N_REP), _full((N_REP, d))]
                _lib.check(L.sgdml_b200_metad_get_bias(H, *map(_p, bias), st), 'metad_get_bias')
                out += [n] + hills + bias
            return [x.tobytes() for x in out]

        # each entry point with arguments valid for it: the call's return code and its outputs, sentinel-filled
        def call(entry, H):
            if entry == 'md_set_state':
                return L.sgdml_b200_md_set_state(H, _p(R0), _p(V0), 7, st), []
            if entry == 'md_get_state':
                o = [_full((N_REP, d)), _full(1, np.uint64)]
                return L.sgdml_b200_md_get_state(H, _p(o[0]), None, None, None, _p(o[1]), st), o
            if entry == 'md_run':
                o = [_full((2, N_REP, d)), _full((2, N_REP))]
                return L.sgdml_b200_md_run(H, 2, dt, gamma, kT, 1, 1, _p(o[0]), None, _p(o[1]), None, st), o
            if entry == 'remd_run':
                kTs = np.array([kT, 1.5 * kT, 2.0 * kT])
                o = [_full((2, N_REP, d)), _full((2, N_REP), np.int32), _full((2, 2), np.int64)]
                return L.sgdml_b200_remd_run(H, 3, _p(kTs), 2, dt, gamma, 1, 1, 1, _p(o[0]), None, None, None,
                                             _p(o[1]), None, _p(o[2]), None, st), o
            if entry == 'neb_fire':
                o = [_full(2, np.int64), _full(2), _full(2, np.int32)]
                return L.sgdml_b200_neb_fire(H, 3, 2, 1e-3, 0.1, 1, 0.01, 0.1, 1.0, _p(o[0]), None, _p(o[1]),
                                             _p(o[2]), st), o
            if entry == 'dimer_fire':
                modes = np.random.default_rng(3).standard_normal((N_REP // 2, d))
                o = [_full(3, np.int64), _full(3), _full(3), _full((3, d))]
                return L.sgdml_b200_dimer_fire(H, _p(modes), 2, 1e-3, 1e-3, np.cos(np.pi / 8), np.sin(np.pi / 8), 0.0,
                                               0.01, 0.1, 1.0, _p(o[0]), None, _p(o[1]), _p(o[2]), None, _p(o[3]),
                                               st), o
            if entry == 'pimd_run':
                o = [_full((2, N_REP, d)), _full((2, N_REP))]
                return L.sgdml_b200_pimd_run(H, 2, dt, kT, 20.0 * kT * dt, gamma, 0.5, 1, 1, _p(o[0]), None, None,
                                             None, _p(o[1]), None, st), o
            if entry in ('relax_fire', 'relax_lbfgs'):
                o = [_full(N_REP, np.int64), _full(N_REP, np.int32), _full(N_REP)]
                if entry == 'relax_fire':
                    rc = L.sgdml_b200_relax_fire(H, 2, 1e-3, 0.01, 0.1, 1.0, *map(_p, o), st)
                else:
                    rc = L.sgdml_b200_relax_lbfgs(H, 2, 1e-3, 0.01, 5, 1e-2, *map(_p, o), st)
                return rc, o
            if entry == 'npt_run':
                o = [_full((2, N_REP, d)), _full((2, N_REP, 9)), _full((2, N_REP))]
                return L.sgdml_b200_npt_run(H, 2, dt, gamma, kT, 0.0, 1e-4, 20.0 * dt, 1, 1, _p(o[0]), None, None,
                                            None, _p(o[1]), _p(o[2]), st), o
            if entry == 'npt_set_cells':
                return L.sgdml_b200_npt_set_cells(H, _p(L0), _p(L0inv), st), []
            if entry == 'npt_get_cells':
                o = [_full((N_REP, 9)), _full((N_REP, 9)), _full((N_REP, 9))]
                return L.sgdml_b200_npt_get_cells(H, *map(_p, o), st), o
            if entry == 'metad_run':
                widths = np.array([0.1])
                o = [_full((2, N_REP, d)), _full((2, N_REP, 1)), _full((2, N_REP))]
                return L.sgdml_b200_metad_run(H, 2, dt, gamma, kT, 1e-4, _p(widths), 1, np.inf, 1, 1, _p(o[0]), None,
                                              None, None, _p(o[1]), _p(o[2]), st), o
            if entry == 'metad_get_hills':
                o = [_full(n_groups, np.int64)]
                return L.sgdml_b200_metad_get_hills(H, _p(o[0]), None, None, None, st), o
            if entry == 'metad_set_hills':
                return L.sgdml_b200_metad_set_hills(H, _p(np.zeros(n_groups, dtype=np.int64)), None, None, None,
                                                    st), []
            if entry == 'metad_get_bias':
                o = [_full((N_REP, 1)), _full(N_REP), _full((N_REP, d))]
                return L.sgdml_b200_metad_get_bias(H, *map(_p, o), st), o
            raise AssertionError(entry)

        for name, H in handles.items():
            _lib.check(L.sgdml_b200_md_set_state(H, _p(R0), _p(V0), 7, st), 'md_set_state')
        wrong = []
        for entry, accepted in ACCEPTS.items():
            for name, H in handles.items():
                kind = kinds[name]
                before = snapshot(H, kind)
                rc, outs = call(entry, H)
                if kind in accepted:
                    if rc != 0:
                        wrong.append((entry, name, 'refused', rc, _lib.last_error()))
                    continue
                after = snapshot(H, kind)
                untouched = all(np.all(o == _full(o.shape, o.dtype)) for o in outs)
                if rc > -1000 or not untouched or after != before:
                    wrong.append((entry, name, 'accepted', rc, untouched, after == before))
        assert not wrong, wrong
    finally:
        for H in handles.values():
            assert L.sgdml_b200_md_destroy(H) == 0
