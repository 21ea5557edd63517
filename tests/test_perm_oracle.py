"""CPU: the permutation search (oracle/perm.py, the host steps of sgdml_b200/perm.py, the assignment solver built for the
host) against what the unmodified reference recorded in tests/golden/perms/ (make_golden_perms.py), the C ABI's
argument checks, and the drop-in without a device."""

import ctypes
import glob
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import scipy.optimize
from scipy.sparse import csr_matrix

from conftest import GOLDEN_DIR, ROOT

from oracle import perm as operm

PERM_DIR = os.path.join(GOLDEN_DIR, 'perms')
CASES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(PERM_DIR, '*.npz')))


def load_case(name):
    with np.load(os.path.join(PERM_DIR, name + '.npz'), allow_pickle=False) as f:
        g = {k: f[k] for k in f.files}
    g['lat_and_inv'] = (g['lattice'], np.linalg.inv(g['lattice'])) if np.any(g['lattice']) else None
    return g


def test_fixture_set_is_complete():
    assert CASES == ['n21_s6_species', 'n9_s6', 'pbc_n9_s6', 'salvage_n12']
    assert int(load_case('n21_s6_species')['n_penalty_matters']) > 0
    assert len(set(load_case('n21_s6_species')['z'].tolist())) > 1
    assert bool(load_case('salvage_n12')['salvaged']) and load_case('pbc_n9_s6')['lat_and_inv'] is not None


@pytest.mark.parametrize('name', CASES)
def test_planted_generator_reproduces_fixture_inputs(name):
    from sgdml_b200 import synth

    g = load_case(name)
    R, z, idx = synth.planted_symmetry_geometries(int(g['n_atoms']), int(g['n_geos']), g['planted_group'],
                                                  int(g['seed']), float(g['spread']))
    assert np.array_equal(R, g['R']) and np.array_equal(z, g['z']) and np.array_equal(idx, g['g'])
    # z is constant on the group's orbits, and geometry k is the base geometry relabelled by its group element
    assert all(np.array_equal(z[p], z) for p in g['planted_group'])
    r0 = synth.base_geometry(int(g['n_atoms']))
    assert np.max(np.abs(R - r0[g['planted_group'][idx]])) < 6 * float(g['spread'])


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference(name):
    g = load_case(name)
    N = int(g['n_atoms'])
    pair_perms, match_cost = operm.bipartite_match(g['R'], g['z'], g['lat_and_inv'])
    dense = match_cost.toarray()
    off = ~np.eye(dense.shape[0], dtype=bool)
    assert np.all(np.isinf(np.diag(dense)))
    assert np.max(np.abs(dense[off] - g['match_cost'][off]) / np.abs(g['match_cost'][off])) < 1e-12
    keys = sorted(pair_perms)
    assert np.array_equal(np.array(keys).reshape(-1, 2), g['pair_keys'])
    assert np.array_equal(np.array([pair_perms[k] for k in keys]).reshape(-1, N), g['pair_perms'])
    match_perms = operm.sync_perm_mat(pair_perms, match_cost, N)
    assert np.array_equal(match_perms, g['match_perms'])
    group, info = operm.find_perms(g['R'], g['z'], g['lat_and_inv'])
    assert info['salvaged'] == bool(g['salvaged'])
    if bool(g['group_is_none']):
        assert group is None
    else:
        assert group.dtype == g['group'].dtype and np.array_equal(group, g['group'])
        assert sorted(map(tuple, group)) == sorted(map(tuple, g['planted_group']))


def test_host_steps_of_the_engine_match_reference():
    """sync_perm_mat / salvage_subgroup / complete_sym_group of sgdml_b200.perm are integer host code: bit-exact, fed
    with the reference's pairwise results (no device needed)."""
    from sgdml_b200 import perm as eperm

    for name in CASES:
        g = load_case(name)
        N = int(g['n_atoms'])
        pair_perms = {tuple(k): p for k, p in zip(g['pair_keys'].tolist(), g['pair_perms'])}
        match_perms = eperm.sync_perm_mat(pair_perms, csr_matrix(g['match_cost']), N)
        assert np.array_equal(match_perms, g['match_perms'])
        closed = eperm.complete_sym_group(match_perms, n_perms_max=100)
        if bool(g['salvaged']):
            assert closed is None
            assert eperm.complete_sym_group(eperm.salvage_subgroup(match_perms), n_perms_max=100) is None
        else:
            assert closed.dtype == g['group'].dtype and np.array_equal(closed, g['group'])
    g = load_case('salvage_n12')
    for mod in (eperm, operm):
        kept = mod.salvage_subgroup(g['salvage_in'])
        assert np.array_equal(kept, g['salvage_out']) and 0 < len(kept) < len(g['salvage_in'])
        assert np.array_equal(mod.complete_sym_group(kept, n_perms_max=100), g['salvage_closed'])


def test_host_preparation_matches_oracle():
    from sgdml_b200 import perm as eperm

    for name in ('n9_s6', 'pbc_n9_s6'):
        g = load_case(name)
        adj, absv = eperm.prepare(g['R'], g['lat_and_inv'])
        adj_o, v_o = operm.prepare(g['R'], g['lat_and_inv'])
        assert np.array_equal(adj, adj_o) and np.array_equal(absv, np.fabs(v_o))
        assert np.array_equal(adj, np.transpose(adj, (0, 2, 1)))
    g = load_case('pbc_n9_s6')
    assert np.max(operm.prepare(g['R'])[0]) > np.max(operm.prepare(g['R'], g['lat_and_inv'])[0]) + 0.5  # pairs wrap


def test_callbacks_follow_the_reference_protocol():
    from sgdml_b200 import perm as eperm

    seen = []

    def cb(*a, **k):
        seen.append((a, k))

    g = load_case('n9_s6')
    pair_perms = {tuple(k): p for k, p in zip(g['pair_keys'].tolist(), g['pair_perms'])}
    mp = eperm.sync_perm_mat(pair_perms, csr_matrix(g['match_cost']), 9, callback=cb)
    eperm.complete_sym_group(mp, n_perms_max=100, callback=cb)
    assert [a for a, _ in seen] == [(0,), (1,), (0,), (1,)]
    assert seen[0][1]['disp_str'].startswith('Multi-partite') and seen[3][1]['sec_disp_str'] == 'found 6 symmetries'
    seen.clear()
    assert eperm.complete_sym_group(load_case('salvage_n12')['match_perms'], n_perms_max=100, callback=cb) is None
    assert seen[-1][1] == dict(disp_str='Permutation group completion', sec_disp_str='transitive closure has failed',
                               done_with_warning=True)


@pytest.fixture(scope='module')
def lap_host(tmp_path_factory):
    """The solver header of the matching kernel, compiled for the host with a team of one thread."""
    cxx = shutil.which('c++') or shutil.which('g++')
    if cxx is None:
        pytest.skip('no host C++ compiler')
    out = str(tmp_path_factory.mktemp('lap') / 'lap_host.so')
    subprocess.check_call([cxx, '-O2', '-std=c++17', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'sgdml_b200', 'csrc'),
                           os.path.join(ROOT, 'tests', 'perm_host', 'lap_host.cpp'), '-o', out])
    handle = ctypes.CDLL(out)
    handle.lap_host.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_void_p,
                                ctypes.c_void_p]

    def solve(cost, z, penalty):
        n = cost.shape[0]
        buf = np.zeros((n, n | 1))
        buf[:, :n] = cost
        z32 = np.ascontiguousarray(z, dtype=np.int32)
        out = np.full(n, -1, dtype=np.int32)
        rc = handle.lap_host(n, buf.ctypes.data, n | 1, penalty, z32.ctypes.data, out.ctypes.data)
        assert rc == 0 and sorted(out.tolist()) == list(range(n))
        return out

    return solve


def test_host_build_of_the_solver_against_scipy(lap_host):
    rng = np.random.default_rng(5)
    for trial in range(2000):
        n = int(rng.integers(2, 48)) if trial % 100 else int(rng.integers(100, 260))
        kind = trial % 4
        if kind == 0:
            c = rng.standard_normal((n, n))
        elif kind == 1:  # the kernel's kind of cost: minus a product of non-negative matrices
            c = -np.abs(rng.standard_normal((n, n))) @ np.abs(rng.standard_normal((n, n))).T
        elif kind == 2:  # exact ties everywhere
            c = rng.integers(0, 4, (n, n)).astype(np.float64)
        else:  # a planted assignment under noise
            c = -np.eye(n)[rng.permutation(n)] + 1e-3 * rng.standard_normal((n, n))
        z = rng.integers(0, 3, n) if trial % 3 == 0 else np.zeros(n, dtype=np.int64)
        pen = float(np.max(np.abs(c)))
        full = c + (z[:, None] != z[None, :]) * pen
        p = lap_host(c, z, pen)
        rows, ref = scipy.optimize.linear_sum_assignment(full)
        got, want = full[np.arange(n), p].sum(), full[rows, ref].sum()
        assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (trial, n, kind)
        if kind != 2:
            assert np.array_equal(p, ref), (trial, n, kind)


def test_host_build_of_the_solver_returns_a_permutation_for_any_input(lap_host):
    """Bounded loops and a valid permutation whatever the numbers are (the kernel must not depend on its input to end
    or to stay inside its arrays)."""
    rng = np.random.default_rng(6)
    z = np.zeros(9, dtype=np.int64)
    for fill in (np.nan, np.inf, -np.inf, 0.0):
        lap_host(np.full((9, 9), fill), z, fill)
    c = rng.standard_normal((9, 9))
    c[rng.integers(0, 9, 25), rng.integers(0, 9, 25)] = np.nan
    lap_host(c, z, 1.0)
    # exact ties: the lowest column wins, so identical rows come out in index order
    assert lap_host(np.zeros((5, 5)), z[:5], 0.0).tolist() == [0, 1, 2, 3, 4]


def test_c_abi_argument_checks_need_no_device():
    from sgdml_b200 import _lib

    L = _lib.lib()
    M, N = 3, 4
    a = np.zeros((M, N, N))
    z = np.zeros(N, dtype=np.int64)
    cost = np.zeros((M, M))
    ok_pairs = np.array([[0, 1], [1, 2]], dtype=np.int64)

    def call(adj=a, absv=a, zz=z, m=M, n=N, pairs=None, n_pairs=0, out=cost):
        return L.sgdml_b200_bipartite_match(_lib.ptr(adj), _lib.ptr(absv), _lib.ptr(zz), m, n, _lib.ptr(pairs), n_pairs,
                                            _lib.ptr(out), None, None, None)

    ERR_ARG = -1000
    assert call(n=1) == ERR_ARG and 'n_atoms' in _lib.last_error()
    assert call(n=1024) == ERR_ARG
    assert call(m=0) == ERR_ARG and call(m=65536) == ERR_ARG
    assert call(adj=None) == ERR_ARG and call(absv=None) == ERR_ARG and call(zz=None) == ERR_ARG
    assert call(out=None) == ERR_ARG
    for bad in ([[1, 1]], [[2, 1]], [[0, 3]], [[-1, 2]]):
        assert call(pairs=np.array(bad, dtype=np.int64), n_pairs=1) == ERR_ARG, bad
        assert 'pairs' in _lib.last_error()
    assert call(pairs=ok_pairs, n_pairs=-1) == ERR_ARG
    # valid arguments get as far as the device check
    import torch

    if not torch.cuda.is_available():
        assert call(pairs=ok_pairs, n_pairs=2, out=np.zeros(2)) == -1002
        assert call() == -1002
    plan = (ctypes.c_int64 * 5)()
    assert L.sgdml_b200_bipartite_match_plan(1, plan) == ERR_ARG
    assert L.sgdml_b200_bipartite_match_plan(N, None) == ERR_ARG


def test_plan_switches_to_the_slab_from_size_alone():
    from sgdml_b200 import perm as eperm

    for n, path, threads in ((2, 'smem', 32), (21, 'smem', 32), (33, 'smem', 64), (100, 'smem', 128),
                             (112, 'smem', 128), (113, 'slab', 128), (160, 'slab', 256), (1023, 'slab', 256)):
        plan = eperm.match_plan(n)
        assert (plan['path'], plan['threads']) == (path, threads), n
        assert plan['smem_bytes'] <= 227 * 1024
        assert (plan['slab_doubles'] >= n * n) == (path == 'slab')


def _stub_reference(monkeypatch, with_perm):
    class RefTrain(object):
        def create_task(self, *a, **k):
            return 'task'

        def create_task_from_model(self, *a, **k):
            return 'task from model'

        def draw_strat_sample(self, *a, **k):
            return 'sample'

    def ref_find_perms(R, z, lat_and_inv=None, callback=None, max_processes=None):
        return 'reference perms'

    mods = {n: types.ModuleType(n) for n in ('refstub2', 'refstub2.cli', 'refstub2.train')}
    mods['refstub2.cli'].GDMLTrain, mods['refstub2.cli'].GDMLPredict = RefTrain, object
    mods['refstub2.train'].GDMLTrain = RefTrain
    mods['refstub2'].cli, mods['refstub2'].train = mods['refstub2.cli'], mods['refstub2.train']
    if with_perm:
        utils, perm = types.ModuleType('refstub2.utils'), types.ModuleType('refstub2.utils.perm')
        perm.find_perms = ref_find_perms
        utils.perm = perm
        mods['refstub2'].utils = utils
        mods.update({'refstub2.utils': utils, 'refstub2.utils.perm': perm})
    for name, mod in mods.items():
        monkeypatch.setitem(sys.modules, name, mod)
    return mods['refstub2'], ref_find_perms


@pytest.mark.parametrize('with_perm', [False, True])
def test_dropin_leaves_find_perms_alone_without_a_device(monkeypatch, with_perm):
    import sgdml_b200
    from sgdml_b200 import _lib
    from sgdml_b200.integration import install_into_reference

    pkg, ref_find_perms = _stub_reference(monkeypatch, with_perm)
    T, P = install_into_reference(pkg)
    assert pkg.cli.GDMLTrain is T and pkg.cli.GDMLPredict is P
    if with_perm:
        if _lib.lib().sgdml_b200_device_count() < 1:
            assert pkg.utils.perm.find_perms is ref_find_perms
        else:
            assert pkg.utils.perm.find_perms is sgdml_b200.find_perms
    else:
        assert not hasattr(pkg, 'utils')


def test_engine_signatures_equal_the_reference():
    import inspect

    from sgdml_b200 import perm as eperm

    want = {
        'bipartite_match': ['R', 'z', 'lat_and_inv', 'max_processes', 'callback'],
        'sync_perm_mat': ['match_perms_all', 'match_cost', 'n_atoms', 'callback'],
        'salvage_subgroup': ['perms'],
        'complete_sym_group': ['perms', 'n_perms_max', 'disp_str', 'callback'],
        'find_perms': ['R', 'z', 'lat_and_inv', 'callback', 'max_processes'],
    }
    for name, params in want.items():
        assert list(inspect.signature(getattr(eperm, name)).parameters) == params, name
