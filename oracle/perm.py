"""CPU oracle of the permutation search (reference utils/perm.py:53-412) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

NumPy / SciPy restatement, single process, no module state: pairwise matching of the training geometries with
``scipy.optimize.linear_sum_assignment`` (perm.py:53-235), the minimum spanning tree over the match costs and the
permutations on its edges (perm.py:238-259), closure of those under composition with a cap (perm.py:344-381), and the
fallback that drops permutations with conflicting cycles when closure hits the cap (perm.py:263-341, 402-410).
``tests/golden/make_golden_perms.py`` pins it against the unmodified reference (``tests/golden/perms/*.npz``).
"""

import numpy as np
import scipy.optimize
import scipy.spatial.distance
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import minimum_spanning_tree

N_PERMS_MAX = 100  # perm.py:398-400


def pair_distances(r, lat_and_inv=None):
    """Full (N, N) distance matrix of one geometry r (N, 3): SciPy's pdist for a free molecule (perm.py:148), and with
    a cell the minimum-image difference of every pair a < b (perm.py:177-183, utils/desc.py:44-77, 105-107:
    d = r_a - r_b, d -= lat @ around(lat_inv @ d), lattice vectors as columns), mirrored."""
    if lat_and_inv is None:
        return scipy.spatial.distance.squareform(scipy.spatial.distance.pdist(r, 'euclidean'))
    lat, lat_inv = lat_and_inv
    a, b = np.triu_indices(r.shape[0], k=1)
    diff = r[a] - r[b]
    diff = diff - np.around(diff.dot(np.asarray(lat_inv).T)).dot(np.asarray(lat).T)
    d = np.zeros((r.shape[0], r.shape[0]))
    d[a, b] = d[b, a] = np.sqrt(np.sum(diff * diff, axis=-1))
    return d


def spectral_embedding(adj):
    """Eigenvectors of a distance matrix, columns by descending eigenvalue (perm.py:185-186).  np.linalg.eig, not
    eigh: the general solver's vectors are what the reference matches on."""
    w, v = np.linalg.eig(adj)
    return v[:, w.argsort()[::-1]]


def prepare(R, lat_and_inv=None):
    """(adj (M, N, N), v (M, N, N)) of the geometries R (M, N, 3)."""
    M, N = R.shape[:2]
    adj = np.empty((M, N, N))
    v = np.empty((M, N, N))
    for i in range(M):
        adj[i] = pair_distances(R[i], lat_and_inv)
        v[i] = spectral_embedding(adj[i])
    return adj, v


def pair_cost(v_i, v_j, z):
    """Assignment cost of one pair (perm.py:70-71, 97-98)."""
    cost = -np.fabs(v_i).dot(np.fabs(v_j).T)
    cost += (z[:, None] != z[None, :]) * np.max(np.abs(cost))
    return cost


def match_pair(adj_i, adj_j, v_i, v_j, z):
    """(perm, match_cost, has_perm) of one pair (perm.py:61-85)."""
    _, perm = scipy.optimize.linear_sum_assignment(pair_cost(v_i, v_j, z))
    before = np.linalg.norm(adj_i - adj_j)
    after = np.linalg.norm(adj_i[perm][:, perm] - adj_j)
    if after >= before:
        return perm, before, False
    return perm, after, not np.isclose(before, after)


def bipartite_match(R, z, lat_and_inv=None):
    """({(i, j): perm}, match_cost as CSR with an infinite diagonal) over all pairs i < j (perm.py:90-235)."""
    z = np.asarray(z)
    M = R.shape[0]
    adj, v = prepare(R, lat_and_inv)
    cost = np.zeros((M, M))
    perms = {}
    for i in range(M):
        for j in range(i + 1, M):
            perm, cost[i, j], keep = match_pair(adj[i], adj[j], v[i], v[j], z)
            if keep:
                perms[i, j] = perm
    cost = cost + cost.T
    cost[np.diag_indices_from(cost)] = np.inf
    return perms, csr_matrix(cost)


def tree_edges(match_cost):
    """Edges (row, col) of the minimum spanning tree of the match costs, in the order its nonzeros are listed."""
    tree = minimum_spanning_tree(match_cost.copy())
    return list(zip(*tree.nonzero()))


def sync_perm_mat(match_perms_all, match_cost, n_atoms):
    """Identity plus the permutations found on the spanning tree's edges, unique and sorted (perm.py:238-259)."""
    rows = [np.arange(n_atoms, dtype=int)]
    for edge in tree_edges(match_cost):
        perm = match_perms_all.get(edge)
        if perm is not None:
            rows.append(np.asarray(perm, dtype=int))
    return np.unique(np.array(rows, dtype=int), axis=0)


def cycles(perm):
    """Disjoint cycles of a permutation, fixed points as cycles of length one."""
    seen = np.zeros(len(perm), dtype=bool)
    out = []
    for start in range(len(perm)):
        if seen[start]:
            continue
        cyc, a = [], start
        while not seen[a]:
            seen[a] = True
            cyc.append(a)
            a = int(perm[a])
        out.append(cyc)
    return out


def salvage_subgroup(perms):
    """Keeps the permutations none of whose cycles (longer than one) shares an atom with a longer cycle of any of the
    permutations (perm.py:289-341)."""
    long_cycles = [[set(c) for c in cycles(p) if len(c) > 1] for p in perms]
    every = [c for cs in long_cycles for c in cs]
    keep = [
        k
        for k, cs in enumerate(long_cycles)
        if not any(len(c) < len(o) and not c.isdisjoint(o) for c in cs for o in every)
    ]
    return perms[keep, :]


def complete_sym_group(perms, n_perms_max=None):
    """Closure under composition, new elements appended in the reference's order; None once n_perms_max rows are
    reached (perm.py:344-381)."""
    perms = np.asarray(perms)
    grew = True
    while grew:
        grew = False
        n = perms.shape[0]
        for i in range(n):
            for j in range(n):
                new = perms[i, perms[j]]
                if not (new == perms).all(axis=1).any():
                    grew = True
                    perms = np.vstack((perms, new))
                    if n_perms_max is not None and perms.shape[0] == n_perms_max:
                        return None
    return perms


def find_perms(R, z, lat_and_inv=None):
    """perm.py:384-412.  Returns (group, info) with info = dict(match_perms=..., salvaged=bool)."""
    n_atoms = R.shape[1]
    match_perms_all, match_cost = bipartite_match(R, z, lat_and_inv)
    match_perms = sync_perm_mat(match_perms_all, match_cost, n_atoms)
    group = complete_sym_group(match_perms, N_PERMS_MAX)
    salvaged = group is None
    if salvaged:
        group = complete_sym_group(salvage_subgroup(match_perms), N_PERMS_MAX)
    return group, dict(match_perms=match_perms, salvaged=salvaged)
