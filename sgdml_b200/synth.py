"""Seeded synthetic molecules, labels and permutation groups (SURVEY.md section 8d).

No datasets are available offline (the reference downloads them, sgdml/get.py:46-49),
so every test and benchmark runs on these generators.  Host-side NumPy only; nothing
here is on the hot path.
"""

import numpy as np


def base_geometry(n_atoms, seed=12345):
    """First N points of a ceil(N^(1/3))^3 cubic grid (1.5 A spacing) + U(-0.1, 0.1) jitter."""
    rng = np.random.default_rng(seed + 7919 * n_atoms)
    k = int(np.ceil(n_atoms ** (1.0 / 3.0) - 1e-9))
    grid = np.array([(x, y, z) for x in range(k) for y in range(k) for z in range(k)], dtype=np.float64)
    r0 = 1.5 * grid[:n_atoms] + rng.uniform(-0.1, 0.1, size=(n_atoms, 3))
    return r0


def geometries(n_atoms, n_geos, seed, spread=0.05, r0=None):
    """R_k = r0 + spread * N(0,1).  Returns (n_geos, N, 3).  Train: seed 0; query: seed 1."""
    if r0 is None:
        r0 = base_geometry(n_atoms)
    rng = np.random.default_rng(seed)
    return r0[None] + spread * rng.standard_normal((n_geos, n_atoms, 3))


def toy_pes(R):
    """E = sum_{a<b} 1/d_ab, F_a = sum_b (r_a - r_b)/d_ab^3  (F = -dE/dr)."""
    R = np.asarray(R, dtype=np.float64)
    diff = R[:, :, None, :] - R[:, None, :, :]
    d = np.sqrt(np.sum(diff * diff, axis=-1))
    n = R.shape[1]
    iu = np.triu_indices(n, 1)
    E = np.sum(1.0 / d[:, iu[0], iu[1]], axis=1)
    with np.errstate(divide='ignore', invalid='ignore'):
        w = 1.0 / d**3
    w[:, np.arange(n), np.arange(n)] = 0.0
    F = np.sum(diff * w[..., None], axis=2)
    return E, F


def close_group(gens, n_atoms, max_size=100000):
    """Close a set of generator permutations under composition (breadth first).
    Identity first; deterministic order."""
    ident = tuple(range(n_atoms))
    seen = {ident: 0}
    order = [ident]
    frontier = [ident]
    gens = [tuple(int(x) for x in g) for g in gens]
    while frontier:
        nxt = []
        for p in frontier:
            for g in gens:
                q = tuple(p[g[a]] for a in range(n_atoms))
                if q not in seen:
                    seen[q] = len(order)
                    order.append(q)
                    nxt.append(q)
                    if len(order) > max_size:
                        raise ValueError('group closure exceeds max_size')
        frontier = nxt
    return np.array(order, dtype=np.int64)


def rotor_swap_group(n_atoms, n_rotors=1, n_swaps=1):
    """Direct product of 3-cycles on disjoint atom triples ("methyl rotors") and 2-swaps
    on disjoint pairs: S = 3^n_rotors * 2^n_swaps."""
    need = 3 * n_rotors + 2 * n_swaps
    if need > n_atoms:
        raise ValueError('not enough atoms for the requested generators')
    gens = []
    at = 0
    for _ in range(n_rotors):
        g = list(range(n_atoms))
        g[at], g[at + 1], g[at + 2] = at + 1, at + 2, at
        gens.append(g)
        at += 3
    for _ in range(n_swaps):
        g = list(range(n_atoms))
        g[at], g[at + 1] = at + 1, at
        gens.append(g)
        at += 2
    if not gens:
        return np.arange(n_atoms, dtype=np.int64)[None, :]
    return close_group(gens, n_atoms)


def c60_geometry(radius=3.55):
    """Ideal truncated icosahedron (buckyball C60): the 60 vertices are the even (cyclic)
    permutations of (0, +-1, +-3phi), (+-1, +-(2+phi), +-2phi), (+-phi, +-2, +-(2phi+1)),
    scaled to the given radius [A] (SURVEY.md section 8d, config 5)."""
    phi = (1.0 + np.sqrt(5.0)) / 2.0
    base = []
    for a, b, c in [(0.0, 1.0, 3 * phi), (1.0, 2 + phi, 2 * phi), (phi, 2.0, 2 * phi + 1)]:
        for sa in ((1,) if a == 0 else (1, -1)):
            for sb in (1, -1):
                for sc in (1, -1):
                    base.append((sa * a, sb * b, sc * c))
    pts = []
    for v in base:
        for k in range(3):  # cyclic coordinate permutations
            pts.append((v[(0 + k) % 3], v[(1 + k) % 3], v[(2 + k) % 3]))
    r0 = np.array(sorted(set(pts)), dtype=np.float64)
    assert r0.shape == (60, 3)
    return r0 * (radius / np.linalg.norm(r0[0]))


def icosahedral_group(r0=None):
    """The 120 atom permutations of the full icosahedral point group I_h acting on the C60
    vertices: the group is generated from a 2-fold, a 3-fold and a 5-fold rotation plus the
    inversion, closed under multiplication, and every 3x3 matrix is turned into a permutation by
    nearest-atom matching.  Identity first."""
    if r0 is None:
        r0 = c60_geometry()
    phi = (1.0 + np.sqrt(5.0)) / 2.0
    c2 = np.diag([-1.0, -1.0, 1.0])
    c3 = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])  # x -> y -> z -> x
    ax = np.array([0.0, 1.0, phi]) / np.sqrt(1 + phi * phi)  # a 5-fold axis (icosahedron vertex)
    th = 2 * np.pi / 5
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    c5 = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)
    gens = [c2, c3, c5, -np.eye(3)]
    mats = [np.eye(3)]
    keys = {tuple(np.round(np.eye(3), 6).ravel())}
    frontier = [np.eye(3)]
    while frontier:
        nxt = []
        for A in frontier:
            for G in gens:
                B = G @ A
                k = tuple(np.round(B, 6).ravel() + 0.0)
                if k not in keys:
                    keys.add(k)
                    mats.append(B)
                    nxt.append(B)
        frontier = nxt
        if len(mats) > 120:
            raise ValueError('generators do not close into I_h')
    assert len(mats) == 120
    perms = []
    for A in mats:
        moved = r0 @ A.T
        d = np.linalg.norm(moved[:, None, :] - r0[None, :, :], axis=-1)
        p = np.argmin(d, axis=1)
        assert np.all(d[np.arange(60), p] < 1e-6) and len(set(p.tolist())) == 60
        perms.append(p)
    return np.array(perms, dtype=np.int64)


# name -> (n_atoms, n_train, n_rotors, n_swaps, sig): BASELINE.json configs with the
# synthetic defaults fixed in SURVEY.md section 8d.
CONFIGS = {
    'ethanol': dict(n_atoms=9, n_train=200, n_rotors=1, n_swaps=1, sig=20),  # cfg 1, S=6
    'aspirin': dict(n_atoms=21, n_train=1000, n_rotors=1, n_swaps=1, sig=20),  # cfg 2, S=6
    'ac-ala3-nhme': dict(n_atoms=42, n_train=2000, n_rotors=5, n_swaps=0, sig=50),  # cfg 3, S=243
    'synthetic100': dict(n_atoms=100, n_train=5000, n_rotors=1, n_swaps=2, sig=50),  # cfg 4, S=12
    'c60': dict(n_atoms=60, n_train=3000, group='ih', sig=50),  # cfg 5, S=120 (I_h on the ideal buckyball)
}


def config_perms_and_r0(name):
    """(perms, base geometry or None) of a named config."""
    cfg = CONFIGS[name]
    if cfg.get('group') == 'ih':
        r0 = c60_geometry()
        return icosahedral_group(r0), r0
    return rotor_swap_group(cfg['n_atoms'], cfg['n_rotors'], cfg['n_swaps']), None


def make_task(n_atoms, n_train, perms, sig, lam=1e-10, seed=0, use_E=True, r0=None):
    """A task dict with the keys GDMLTrain.train reads (reference sgdml/train.py:507-524)."""
    R = geometries(n_atoms, n_train, seed, r0=r0)
    E, F = toy_pes(R)
    return {
        'type': 't',
        'code_version': 'synthetic',
        'dataset_name': 'synthetic_%d' % n_atoms,
        'dataset_theory': 'toy_inverse_distance',
        'z': np.arange(1, n_atoms + 1, dtype=np.int64) % 9 + 1,
        'R_train': R,
        'F_train': F,
        'E_train': E,
        'idxs_train': np.arange(n_train, dtype=np.int64),
        'md5_train': b'0' * 32,
        'idxs_valid': np.arange(0, dtype=np.int64),
        'md5_valid': b'0' * 32,
        'sig': sig,
        'lam': lam,
        'use_E': use_E,
        'use_E_cstr': False,
        'use_sym': True,
        'perms': np.asarray(perms, dtype=np.int64),
    }


def make_config_task(name, n_train=None, seed=0):
    cfg = dict(CONFIGS[name])
    if n_train is not None:
        cfg['n_train'] = n_train
    perms, r0 = config_perms_and_r0(name)
    return make_task(cfg['n_atoms'], cfg['n_train'], perms, cfg['sig'], seed=seed, r0=r0)


def random_model(n_atoms, n_train, perms, sig, seed=0, alpha_scale=1.0, r0=None):
    """A model dict with random (not trained) coefficients -- for predictor benchmarks
    at sizes where training would be the dominant cost.  Same key layout as
    GDMLTrain.create_model (reference sgdml/train.py:793-830)."""
    from .desc import Desc, tril_perms_lin

    R = geometries(n_atoms, n_train, seed, r0=r0).reshape(n_train, -1)
    rng = np.random.default_rng(seed + 99)
    alphas = alpha_scale * rng.standard_normal(n_train * 3 * n_atoms)
    desc = Desc(n_atoms)
    R_desc, R_d_desc = desc.from_R(R)
    if n_train == 1:
        R_desc, R_d_desc = R_desc[None], R_d_desc[None]
    perms = np.asarray(perms, dtype=np.int64)
    return {
        'type': 'm',
        'code_version': 'synthetic',
        'dataset_name': 'synthetic_%d' % n_atoms,
        'dataset_theory': 'random_alphas',
        'solver_name': 'none',
        'z': np.arange(1, n_atoms + 1, dtype=np.int64) % 9 + 1,
        'R_desc': R_desc.T.copy(),
        'R_d_desc_alpha': desc.d_desc_dot_vec(R_d_desc, alphas.reshape(n_train, -1)),
        'alphas_F': alphas,
        'c': 0.0,
        'std': 1.0,
        'sig': sig,
        'lam': 1e-10,
        'perms': perms,
        'tril_perms_lin': tril_perms_lin(perms),
        'use_E': True,
    }


def orbit_species(perms, palette=(1, 6, 7, 8)):
    """Atomic numbers that are constant on the orbits of a permutation group (perms (S, N)), as a molecule's symmetry
    requires: every orbit with more than one atom gets one species, the atoms the group leaves alone cycle through the
    palette."""
    perms = np.asarray(perms, dtype=np.int64)
    n_atoms = perms.shape[1]
    orbit = np.min(perms, axis=0)  # the lowest atom each atom is mapped to: one label per orbit
    z = np.empty(n_atoms, dtype=np.int64)
    for a in range(n_atoms):
        moved = np.count_nonzero(orbit == orbit[a]) > 1
        z[a] = palette[(orbit[a] + (1 if moved else 0)) % len(palette)]
    return z


def planted_symmetry_geometries(n_atoms, n_geos, perms, seed, spread=0.005, r0=None):
    """Geometries that are related by the permutations of a given group (`rotor_swap_group`, `close_group`), which
    `geometries` never produces: R_k = r0[g_k] + spread * N(0, 1) with g_k drawn uniformly (seeded) from `perms`.
    Geometry k is the base geometry with its atoms relabelled by g_k -- what a trajectory of a molecule with rotating
    methyl groups looks like to a permutation search -- so geometries i and j are related by g_i^-1 g_j (atom a of j sits
    where atom g_i^-1[g_j[a]] of i sits), a search finds that element or its inverse, and the closure of what it finds
    is the group.  The base geometry needs no symmetry of its own.  The spread is small on purpose: the spectral
    matching of perm.py loses pairs once the noise mixes close-lying eigenvectors (0.02 already does at 9 atoms).  Returns (R (n_geos, N, 3), z (N,) constant on the group's orbits, g (n_geos,) the index of
    each geometry's group element).

    How many geometries: a spanning tree over the geometries carries a generating set once every one of the S elements
    has been drawn (the products of the matches along the tree's paths then reach every element); a draw of n_geos
    misses some element with probability at most S (1 - 1/S)^n_geos, about S exp(-n_geos / S): 7 % at n_geos = 4 S for
    S = 6, below 1 % from 6 S.  Fewer elements usually still generate the group, but nothing guarantees it."""
    perms = np.asarray(perms, dtype=np.int64)
    if r0 is None:
        r0 = base_geometry(n_atoms)
    rng = np.random.default_rng(seed)
    g = rng.integers(0, perms.shape[0], size=n_geos)
    noise = rng.standard_normal((n_geos, n_atoms, 3))
    R = r0[perms[g]] + spread * noise
    return R, orbit_species(perms), g
