"""Generates tests/golden/perms/*.npz by running the UNMODIFIED reference's permutation search (stefanch/sGDML v1.0.3,
sgdml/utils/perm.py: bipartite_match, sync_perm_mat, find_perms) on seeded planted-symmetry datasets
(sgdml_b200.synth.planted_symmetry_geometries).  Needs a copy of the reference package under baseline/_ref (or on
PYTHONPATH) and no GPU:

    PYTHONPATH=baseline/_ref:. python tests/golden/make_golden_perms.py

Every fixture holds the generator's arguments and the geometries they give (tests regenerate them from the seed and
compare), z, the cell if any, the planted group, and from the reference: the dense symmetric match-cost matrix, the
pairs for which a permutation was kept with those permutations, the permutations on the spanning tree after
synchronisation, whether closure hit the cap of 100, and the final group.

    n9_s6           9 atoms, methyl rotor x swap (S = 6), 30 geometries
    n21_s6_species  21 atoms, S = 6, four species, noise 0.02: for some pairs the optimal assignment changes when the
                    species penalty (perm.py:71, 97-98) is left out (counted in `n_penalty_matters`)
    pbc_n9_s6       the 9-atom case in a 4 A cubic cell, where most pair distances wrap
    salvage_n12     S_3 on each of three atom triples (S = 216 > 100): closure gives up and the salvage path
                    (perm.py:289-341, 402-410) runs.  The reference keeps a pair's permutation only when applying it
                    the other way round (perm.py:75-76) still lowers the mismatch, so the spanning tree carries
                    involutions only, none of them is dropped, the second closure fails too and the result is None.
                    The fixture therefore also holds a hand-made set with clashing cycles (`salvage_in`) and what the
                    reference's salvage_subgroup and complete_sym_group make of it (`salvage_out`, `salvage_closed`).
"""

import importlib.util
import os
import sys

import numpy as np
import scipy.optimize
from scipy.spatial.distance import pdist, squareform

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'baseline', '_ref'))

_spec = importlib.util.spec_from_file_location('synth', os.path.join(ROOT, 'sgdml_b200', 'synth.py'))
synth = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(synth)

import sgdml  # noqa: E402  (the reference)
from sgdml.utils import perm as rperm  # noqa: E402

assert sgdml.__version__ == '1.0.3'


def s3_cubed(n_atoms):
    gens = []
    for t in range(3):
        rot = list(range(n_atoms))
        rot[3 * t], rot[3 * t + 1], rot[3 * t + 2] = 3 * t + 1, 3 * t + 2, 3 * t
        swap = list(range(n_atoms))
        swap[3 * t], swap[3 * t + 1] = 3 * t + 1, 3 * t
        gens += [rot, swap]
    return synth.close_group(gens, n_atoms)


CASES = {
    'n9_s6': dict(n_atoms=9, n_geos=30, seed=11, group=('rotor_swap', 1, 1), cell=0.0),
    'n21_s6_species': dict(n_atoms=21, n_geos=26, seed=12, group=('rotor_swap', 1, 1), cell=0.0, spread=0.02),
    'pbc_n9_s6': dict(n_atoms=9, n_geos=30, seed=13, group=('rotor_swap', 1, 1), cell=4.0),
    'salvage_n12': dict(n_atoms=12, n_geos=40, seed=14, group=('s3_cubed',), cell=0.0),
}


def make(name, cfg):
    N, M = cfg['n_atoms'], cfg['n_geos']
    group = s3_cubed(N) if cfg['group'][0] == 's3_cubed' else synth.rotor_swap_group(N, *cfg['group'][1:])
    spread = cfg.get('spread', 0.005)
    R, z, g = synth.planted_symmetry_geometries(N, M, group, cfg['seed'], spread)
    lat_and_inv = None
    lattice = np.zeros((3, 3))
    if cfg['cell'] > 0:
        lattice = cfg['cell'] * np.eye(3)
        lat_and_inv = (lattice, np.linalg.inv(lattice))

    pair_perms, match_cost = rperm.bipartite_match(R, z, lat_and_inv=lat_and_inv, max_processes=1)
    dense = match_cost.toarray()
    keys = sorted(pair_perms)
    match_perms = rperm.sync_perm_mat(pair_perms, match_cost.copy(), N)
    closed = rperm.complete_sym_group(match_perms, n_perms_max=100)
    final = rperm.find_perms(R, z, lat_and_inv=lat_and_inv, max_processes=1)
    salvaged = closed is None
    if not salvaged:
        assert np.array_equal(closed, final)

    # pairs whose optimal assignment depends on the species penalty
    n_matter = 0
    same = z[:, None] != z[None, :]
    vs = []
    for i in range(M if lat_and_inv is None else 0):  # free molecules only
        w, v = np.linalg.eig(squareform(pdist(R[i])))
        vs.append(np.fabs(v[:, w.argsort()[::-1]]))
    for i in range(len(vs)):
        for j in range(i + 1, len(vs)):
            cost = -vs[i].dot(vs[j].T)
            p0 = scipy.optimize.linear_sum_assignment(cost)[1]
            p1 = scipy.optimize.linear_sum_assignment(cost + same * np.max(np.abs(cost)))[1]
            n_matter += not np.array_equal(p0, p1)

    out = dict(
        n_atoms=N, n_geos=M, seed=cfg['seed'], spread=spread, group_kind=np.array(cfg['group'][0]),
        group_args=np.array(cfg['group'][1:], dtype=np.int64), R=R, z=z, g=g, lattice=lattice,
        planted_group=group, match_cost=dense, pair_keys=np.array(keys, dtype=np.int64).reshape(-1, 2),
        pair_perms=np.array([pair_perms[k] for k in keys], dtype=np.int64).reshape(-1, N),
        match_perms=match_perms, salvaged=salvaged, group_is_none=final is None,
        group=final if final is not None else np.zeros((0, N), dtype=np.int64), n_penalty_matters=n_matter,
    )
    if salvaged:
        # identity, a 3-cycle, a swap inside it (dropped), a disjoint swap, a 4-cycle, its square (two swaps inside it:
        # dropped), a swap + 3-cycle that are disjoint from each other but not from the rest
        cyc = np.array([
            [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], [1, 2, 0, 3, 4, 5, 6, 7, 8, 9, 10, 11],
            [1, 0, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11], [0, 1, 2, 4, 3, 5, 6, 7, 8, 9, 10, 11],
            [0, 1, 2, 3, 4, 6, 7, 8, 5, 9, 10, 11], [0, 1, 2, 3, 4, 7, 8, 5, 6, 9, 10, 11],
            [0, 1, 2, 4, 3, 5, 6, 7, 8, 10, 11, 9], [0, 1, 2, 3, 4, 5, 6, 7, 8, 10, 9, 11],
        ])
        out['salvage_in'] = cyc
        out['salvage_out'] = rperm.salvage_subgroup(cyc)
        out['salvage_closed'] = rperm.complete_sym_group(out['salvage_out'], n_perms_max=100)
        print('salvage check: kept', len(out['salvage_out']), 'of', len(cyc), '-> closed', len(out['salvage_closed']))
    os.makedirs(os.path.join(HERE, 'perms'), exist_ok=True)
    np.savez_compressed(os.path.join(HERE, 'perms', name + '.npz'), **out)
    planted = final is not None and sorted(map(tuple, final)) == sorted(map(tuple, group))
    print('%-16s pairs with a permutation %4d / %4d, tree perms %3d, salvaged %s, group %s, planted found %s, '
          'penalty matters for %d pairs' % (name, len(keys), M * (M - 1) // 2, len(match_perms), salvaged,
                                            None if final is None else final.shape[0], planted, n_matter))


if __name__ == '__main__':
    for name, cfg in CASES.items():
        if len(sys.argv) == 1 or name in sys.argv[1:]:
            make(name, cfg)
