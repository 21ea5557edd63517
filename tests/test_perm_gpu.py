"""GPU: the pairwise matching kernel (sgdml_b200_bipartite_match) against the oracle (oracle/perm.py: SciPy's
linear_sum_assignment) and the reference's recorded results (tests/golden/perms/), in both cost-matrix placements
(shared memory up to 112 atoms, global slab above), and sgdml_b200.perm.find_perms end to end."""

import numpy as np
import pytest
import scipy.optimize

from conftest import rel_err
from test_perm_oracle import CASES, load_case

from oracle import perm as operm

pytestmark = pytest.mark.gpu


def _inputs(N, M, seed, n_species):
    from sgdml_b200 import perm as eperm
    from sgdml_b200 import synth

    R = synth.geometries(N, M, seed)
    z = np.arange(N, dtype=np.int64) % n_species + 1
    adj, absv = eperm.prepare(R)
    return adj, absv, z


def _check_pairs(adj, absv, z, pairs, cost, perms, has, exact):
    """Every row a permutation; optimal on the oracle's cost matrix (whatever the tie-breaking); the scores and the
    keep decision as perm.py:75-85 computes them from that permutation; with `exact`, SciPy's permutation itself."""
    N = adj.shape[1]
    for k, (i, j) in enumerate(pairs):
        p = perms[k]
        assert sorted(p.tolist()) == list(range(N)), (i, j)
        c = operm.pair_cost(absv[i], absv[j], z)
        rows, ref = scipy.optimize.linear_sum_assignment(c)
        got, want = c[np.arange(N), p].sum(), c[rows, ref].sum()
        assert abs(got - want) <= 1e-12 * abs(want), (i, j, got, want)
        if exact:
            assert np.array_equal(p, ref), (i, j)
        before = np.linalg.norm(adj[i] - adj[j])
        after = np.linalg.norm(adj[i][p][:, p] - adj[j])
        assert abs(cost[k] - min(before, after)) <= 1e-12 * min(before, after), (i, j)
        assert bool(has[k]) == bool(after < before and not np.isclose(before, after)), (i, j)


@pytest.mark.parametrize('n_species', [1, 3])
@pytest.mark.parametrize('N,M,path', [(2, 40, 'smem'), (3, 40, 'smem'), (9, 30, 'smem'), (21, 24, 'smem'),
                                      (33, 16, 'smem'), (60, 10, 'smem'), (100, 8, 'smem'), (160, 6, 'slab'),
                                      (240, 6, 'slab')])
def test_all_pairs_against_oracle(N, M, path, n_species):
    from sgdml_b200 import perm as eperm

    assert eperm.match_plan(N)['path'] == path
    adj, absv, z = _inputs(N, M, 100 + N, n_species)
    cost, perms, has = eperm.match_pairs(adj, absv, z, want_perms=True)
    iu = np.triu_indices(M, k=1)
    assert np.all(cost[np.tril_indices(M)] == 0.0)  # only the upper triangle is written
    _check_pairs(adj, absv, z, list(zip(*iu)), cost[iu], perms, has, exact=False)


@pytest.mark.parametrize('name', CASES)
def test_fixture_pairs_equal_scipy_and_reference(name):
    from sgdml_b200 import perm as eperm

    g = load_case(name)
    adj, absv = eperm.prepare(g['R'], g['lat_and_inv'])
    M = adj.shape[0]
    cost, perms, has = eperm.match_pairs(adj, absv, g['z'], want_perms=True)
    iu = np.triu_indices(M, k=1)
    _check_pairs(adj, absv, g['z'], list(zip(*iu)), cost[iu], perms, has, exact=True)
    assert np.max(np.abs(cost[iu] - g['match_cost'][iu]) / g['match_cost'][iu]) < 1e-12
    keys = np.stack(iu, axis=1)[has]
    assert np.array_equal(keys, g['pair_keys'])
    assert np.array_equal(perms[has], g['pair_perms'])


@pytest.mark.parametrize('N,M', [(21, 14), (160, 6)])
def test_pair_list_repeat_and_device_pointers_are_bit_identical(N, M):
    import torch

    from sgdml_b200 import perm as eperm

    adj, absv, z = _inputs(N, M, 7, 2)
    cost, perms, has = eperm.match_pairs(adj, absv, z, want_perms=True)
    again = eperm.match_pairs(adj, absv, z, want_perms=True)
    assert np.array_equal(cost, again[0]) and np.array_equal(perms, again[1]) and np.array_equal(has, again[2])

    iu = np.triu_indices(M, k=1)
    order = np.random.default_rng(3).permutation(len(iu[0]))[: max(5, len(iu[0]) // 2)]
    pairs = np.stack(iu, axis=1)[order]
    lcost, lperms, lhas = eperm.match_pairs(adj, absv, z, pairs, want_perms=True)
    assert np.array_equal(lcost, cost[iu][order]) and np.array_equal(lperms, perms[order])
    assert np.array_equal(lhas, has[order])

    dcost, dperms, dhas = eperm.match_pairs(torch.from_numpy(adj).cuda(), torch.from_numpy(absv).cuda(), z, pairs,
                                            want_perms=True)
    assert np.array_equal(dcost, lcost) and np.array_equal(dperms, lperms) and np.array_equal(dhas, lhas)


def test_exact_ties_give_an_optimal_permutation_deterministically():
    from sgdml_b200 import perm as eperm
    from sgdml_b200 import synth

    N = 9
    R = synth.geometries(N, 4, 5)
    R[1] = R[0]  # two identical geometries
    # a geometry with two exactly equivalent atoms: 1 and 2 are mirror images in the plane x = 0 that holds the rest
    R[2, :, 0] = 0.0
    R[2, 1] = [0.7, 0.3, 0.2]
    R[2, 2] = [-0.7, 0.3, 0.2]
    R[3] = R[2]
    z = np.ones(N, dtype=np.int64)
    adj, absv = eperm.prepare(R)
    cost, perms, has = eperm.match_pairs(adj, absv, z, want_perms=True)
    again = eperm.match_pairs(adj, absv, z, want_perms=True)
    assert np.array_equal(perms, again[1]) and np.array_equal(cost, again[0]) and np.array_equal(has, again[2])
    iu = np.triu_indices(4, k=1)
    _check_pairs(adj, absv, z, list(zip(*iu)), cost[iu], perms, has, exact=False)
    assert cost[0, 1] == 0.0 and not has[0]  # identical geometries: nothing to gain


@pytest.mark.parametrize('name', CASES)
def test_find_perms_returns_the_oracle_group(name):
    from sgdml_b200 import perm as eperm

    g = load_case(name)
    progress = []

    def cb(*a, **k):
        if k.get('disp_str') == 'Bi-partite matching':
            progress.append(a)

    group = eperm.find_perms(g['R'], g['z'], lat_and_inv=g['lat_and_inv'], callback=cb, max_processes=4)
    want, _ = operm.find_perms(g['R'], g['z'], g['lat_and_inv'])
    M = int(g['n_geos'])
    assert progress[-1] == (M, M) and all(a[1] == M for a in progress)
    assert [a[0] for a in progress] == sorted(a[0] for a in progress)
    if want is None:
        assert group is None and bool(g['group_is_none'])
        return
    assert sorted(map(tuple, group)) == sorted(map(tuple, want)) == sorted(map(tuple, g['planted_group']))
    assert np.array_equal(group[0], np.arange(int(g['n_atoms'])))


def test_found_group_trains_the_model_of_the_planted_group():
    import sgdml_b200
    from sgdml_b200 import perm as eperm
    from sgdml_b200 import synth

    g = load_case('n9_s6')
    N, M = int(g['n_atoms']), int(g['n_geos'])
    found = eperm.find_perms(g['R'], g['z'])
    assert found.shape == g['planted_group'].shape
    E, F = synth.toy_pes(g['R'])
    Rq = synth.planted_symmetry_geometries(N, 16, g['planted_group'], 99, 0.01)[0].reshape(16, -1)
    forces = []
    for perms in (found, g['planted_group']):
        task = synth.make_task(N, M, perms, 20)
        task.update(R_train=g['R'], E_train=E, F_train=F, z=g['z'])
        model = sgdml_b200.GDMLTrain().train(task)
        forces.append(sgdml_b200.GDMLPredict(model).predict(Rq)[1])
    assert rel_err(forces[0], forces[1]) < 1e-6


def test_non_finite_geometries_are_rejected_on_the_host():
    from sgdml_b200 import perm as eperm

    g = load_case('n9_s6')
    R = g['R'][:4].copy()
    R[2, 0, 0] = np.inf  # never reaches the device
    with pytest.raises((ValueError, np.linalg.LinAlgError)):
        eperm.find_perms(R, g['z'])
