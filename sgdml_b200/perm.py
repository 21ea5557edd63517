"""Permutation discovery: the symmetries of a molecule recovered from its training geometries (reference
sgdml/utils/perm.py:53-412), with the pairwise matching -- one linear assignment problem per pair of geometries, half a
million of them for 1000 training points -- solved on the GPU by ``sgdml_b200_bipartite_match`` (csrc/perm.cu).

Same function names and signatures as the reference module, so a caller switches by import.  Host preparation (pair
distances and the eigenvectors of every distance matrix, perm.py:138-189) uses the reference's own SciPy / LAPACK calls
so that the numbers entering the matching are the same; everything after the matching (spanning tree, group closure,
the fallback when closure fails, perm.py:238-412) is integer code on the host.  There is no CPU fallback for the
matching: without a CUDA device ``bipartite_match`` raises.
"""

import timeit
from functools import partial

import numpy as np
import scipy.spatial.distance
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import minimum_spanning_tree

from . import _lib
from ._lib import check, current_stream, lib, ptr, require_gpu

DONE, NOT_DONE = 1, 0  # the reference's callback protocol (sgdml/__init__.py:31-32)
N_PERMS_MAX = 100  # closure gives up at this many permutations (perm.py:397-400)


def match_plan(n_atoms):
    """How the matching kernel runs at this molecule size: dict(path='smem' | 'slab', threads, smem_bytes,
    slab_doubles, ctas_per_sm).  Host only."""
    out = (_lib.C.c_int64 * 5)()
    check(lib().sgdml_b200_bipartite_match_plan(int(n_atoms), out), 'bipartite_match_plan')
    return dict(path='slab' if out[0] else 'smem', threads=int(out[1]), smem_bytes=int(out[2]),
                slab_doubles=int(out[3]), ctas_per_sm=int(out[4]))


def pair_distances(r, lat_and_inv=None):
    """(N, N) distance matrix of one geometry (N, 3) as perm.py:147-183 builds it: SciPy's pdist, or with a cell the
    minimum-image difference d = r_a - r_b, d -= lat @ around(lat_inv @ d) of every pair a < b (utils/desc.py:44-77)."""
    if lat_and_inv is None:
        return scipy.spatial.distance.squareform(scipy.spatial.distance.pdist(r, 'euclidean'))
    lat, lat_inv = (np.asarray(x, dtype=np.float64) for x in lat_and_inv)
    n = r.shape[0]
    a, b = np.triu_indices(n, k=1)
    d = r[a] - r[b]
    d = d - np.around(d.dot(lat_inv.T)).dot(lat.T)
    adj = np.zeros((n, n))
    adj[a, b] = adj[b, a] = np.sqrt(np.sum(d * d, axis=-1))
    return adj


def prepare(R, lat_and_inv=None):
    """Inputs of the matching for geometries R (M, N, 3): adj (M, N, N) distance matrices and absv (M, N, N) the
    absolute eigenvectors of each, columns by descending eigenvalue (perm.py:185-186; np.linalg.eig as there, so
    near-degenerate eigenvectors come out as the reference's)."""
    R = np.asarray(R, dtype=np.float64)
    M, N = R.shape[:2]
    adj = np.empty((M, N, N))
    absv = np.empty((M, N, N))
    for i in range(M):
        adj[i] = pair_distances(R[i], lat_and_inv)
        w, v = np.linalg.eig(adj[i])
        absv[i] = np.fabs(v[:, w.argsort()[::-1]])
    return adj, absv


def match_pairs(adj, absv, z, pairs=None, want_perms=False, want_has_perm=True):
    """One call of ``sgdml_b200_bipartite_match``.  adj, absv: (M, N, N) NumPy arrays or CUDA tensors.  pairs: None for
    every i < j, or an (n, 2) integer array.  Returns (match_cost, perms or None, has_perm or None) as NumPy arrays:
    match_cost is (M, M) with the upper triangle filled for all pairs and (n,) for a list; perms (n_pairs, N) int32 and
    has_perm (n_pairs,) bool follow the list, or the row-major order of the pairs i < j."""
    require_gpu()
    M, N = int(adj.shape[0]), int(adj.shape[1])
    assert tuple(adj.shape) == (M, N, N) and tuple(absv.shape) == (M, N, N)
    z = np.ascontiguousarray(z, dtype=np.int64)
    assert z.shape == (N,)
    if pairs is None:
        n_pairs = M * (M - 1) // 2
        cost = np.zeros((M, M))
        pairs_arr = None
    else:
        pairs_arr = np.ascontiguousarray(pairs, dtype=np.int64).reshape(-1, 2)
        n_pairs = pairs_arr.shape[0]
        cost = np.zeros(n_pairs)
    perms = np.empty((n_pairs, N), dtype=np.int32) if want_perms else None
    has = np.zeros(n_pairs, dtype=np.uint8) if want_has_perm else None
    check(
        lib().sgdml_b200_bipartite_match(ptr(adj), ptr(absv), ptr(z), M, N, ptr(pairs_arr), n_pairs, ptr(cost),
                                         ptr(perms), ptr(has), current_stream()),
        'bipartite_match',
    )
    return cost, perms, (has.astype(bool) if has is not None else None)


class MatchPerms(object):
    """The permutations the all-pairs matching found, {(i, j): perm} for the pairs i < j whose permutation lowers the
    mismatch (perm.py:84-85), without holding them: at 370 atoms and 1000 geometries they would take 740 MB of which the
    spanning tree reads at most M - 1 rows.  A permutation is computed when it is asked for, by a pair-list call of
    the same deterministic kernel (bit-identical to what the all-pairs call decided on); ``prefetch`` gets many in one
    call."""

    def __init__(self, adj, absv, z, has_perm):
        self._adj, self._absv, self._z = adj, absv, z
        self._M = adj.shape[0]
        self._has = has_perm
        self._cache = {}

    def _index(self, key):
        i, j = int(key[0]), int(key[1])
        if not (0 <= i < j < self._M):
            return None
        return i * self._M - i * (i + 1) // 2 + (j - i - 1)

    def __contains__(self, key):
        k = self._index(key)
        return k is not None and bool(self._has[k])

    def __len__(self):
        return int(np.count_nonzero(self._has))

    def keys(self):
        iu = np.triu_indices(self._M, k=1)
        return [(int(i), int(j)) for i, j, h in zip(iu[0], iu[1], self._has) if h]

    def prefetch(self, keys):
        todo = sorted({(int(i), int(j)) for i, j in keys if (i, j) in self and (int(i), int(j)) not in self._cache})
        if todo:
            _, perms, _ = match_pairs(self._adj, self._absv, self._z, np.array(todo), want_perms=True,
                                      want_has_perm=False)
            for key, p in zip(todo, perms):
                self._cache[key] = p.astype(int)

    def get(self, key, default=None):
        if key not in self:
            return default
        key = (int(key[0]), int(key[1]))
        if key not in self._cache:
            self.prefetch([key])
        return self._cache[key]

    def __getitem__(self, key):
        p = self.get(key)
        if p is None:
            raise KeyError(key)
        return p


def bipartite_match(R, z, lat_and_inv=None, max_processes=None, callback=None):
    """perm.py:90-235 with the loop over pairs as one kernel launch.  Returns (match_perms_all, match_cost):
    a ``MatchPerms`` and the symmetric (M, M) match costs as CSR with an infinite diagonal.  `max_processes` is accepted
    and ignored: there is no process pool behind a CUDA context."""
    R = np.asarray(R, dtype=np.float64)
    n_train = R.shape[0]
    adj, absv = prepare(R, lat_and_inv)
    if not (np.all(np.isfinite(adj)) and np.all(np.isfinite(absv))):
        raise ValueError('bipartite_match: non-finite pair distances or eigenvectors (check the geometries)')
    z = np.ascontiguousarray(z, dtype=np.int64)

    if callback is not None:
        callback = partial(callback, disp_str='Bi-partite matching')
        callback(0, n_train)
    start = timeit.default_timer()
    cost, _, has = match_pairs(adj, absv, z)
    dur_s = timeit.default_timer() - start
    if callback is not None:
        callback(n_train, n_train, sec_disp_str='took {:.1f} s'.format(dur_s) if dur_s >= 0.1 else '')

    cost = cost + cost.T  # perm.py:230-233
    cost[np.diag_indices_from(cost)] = np.inf
    return MatchPerms(adj, absv, z, has), csr_matrix(cost)


def sync_perm_mat(match_perms_all, match_cost, n_atoms, callback=None):
    """perm.py:238-259: the identity and the permutations on the edges of the minimum spanning tree of the match
    costs, unique rows in sorted order."""
    if callback is not None:
        callback = partial(callback, disp_str='Multi-partite matching (permutation synchronization)')
        callback(NOT_DONE)
    tree = minimum_spanning_tree(match_cost, overwrite=True)
    edges = [(int(i), int(j)) for i, j in zip(*tree.nonzero())]
    if hasattr(match_perms_all, 'prefetch'):
        match_perms_all.prefetch(edges)  # all tree edges in one device call
    rows = [np.arange(n_atoms, dtype=int)]
    for edge in edges:
        p = match_perms_all.get(edge)
        if p is not None:
            rows.append(np.asarray(p, dtype=int))
    perms = np.unique(np.array(rows, dtype=int), axis=0)
    if callback is not None:
        callback(DONE)
    return perms


def _long_cycles(perm):
    """The cycles of a permutation that move atoms, as sets."""
    seen = [False] * len(perm)
    out = []
    for start in range(len(perm)):
        cyc, a = set(), start
        while not seen[a]:
            seen[a] = True
            cyc.add(a)
            a = int(perm[a])
        if len(cyc) > 1:
            out.append(cyc)
    return out


def salvage_subgroup(perms):
    """perm.py:289-341: what is kept when closure fails -- the permutations none of whose cycles shares an atom with a
    longer cycle of any permutation of the set."""
    per_perm = [_long_cycles(p) for p in perms]
    every = [c for cs in per_perm for c in cs]

    def clashes(c):
        return any(len(c) < len(o) and not c.isdisjoint(o) for o in every)

    keep = [k for k, cs in enumerate(per_perm) if not any(clashes(c) for c in cs)]
    return perms[keep, :]


def complete_sym_group(perms, n_perms_max=None, disp_str='Permutation group completion', callback=None):
    """perm.py:344-381: closure under composition, products appended in the order (i, j) finds them; None as soon as
    n_perms_max permutations are reached."""
    if callback is not None:
        callback = partial(callback, disp_str=disp_str)
        callback(NOT_DONE)
    perms = np.asarray(perms)
    known = {tuple(p) for p in perms.tolist()}
    rows = [p for p in perms]
    added = True
    while added:
        added = False
        n = len(rows)
        for i in range(n):
            for j in range(n):
                new = rows[i][rows[j]]
                key = tuple(new.tolist())
                if key not in known:
                    added = True
                    known.add(key)
                    rows.append(new)
                    if n_perms_max is not None and len(rows) == n_perms_max:
                        if callback is not None:
                            callback(DONE, sec_disp_str='transitive closure has failed', done_with_warning=True)
                        return None
    perms = np.array(rows, dtype=perms.dtype)
    if callback is not None:
        callback(DONE, sec_disp_str='found {:d} symmetries'.format(perms.shape[0]))
    return perms


def find_perms(R, z, lat_and_inv=None, callback=None, max_processes=None):
    """perm.py:384-412: all-pairs matching on the GPU, permutations on the spanning tree, closure; if closure reaches
    100 permutations, closure of the salvaged subset instead (which may fail too: None)."""
    n_atoms = R.shape[1]
    match_perms_all, match_cost = bipartite_match(R, z, lat_and_inv, max_processes, callback=callback)
    match_perms = sync_perm_mat(match_perms_all, match_cost, n_atoms, callback=callback)
    group = complete_sym_group(match_perms, n_perms_max=N_PERMS_MAX, callback=callback)
    if group is None:
        group = complete_sym_group(salvage_subgroup(match_perms), n_perms_max=N_PERMS_MAX,
                                   disp_str='Closure disaster recovery', callback=callback)
    return group
