"""NumPy restatement of the harmonic vibrational analysis (sgdml_b200/vib.py, csrc/vib.cu): mass weighting, the rigid
basis and the projection that moves it to the top of the spectrum, unit conversion, HarmonicThermo-style thermochemistry
and the Vineyard rate.  Constants are CODATA 2014, as ASE's units."""

import math

import numpy as np

E_CHARGE, AMU, HPLANCK, C_LIGHT, K_B = 1.6021766208e-19, 1.660539040e-27, 6.626070040e-34, 299792458.0, 1.38064852e-23
HBAR = 1.054571800e-34
KB_EV = K_B / E_CHARGE
EV_PER_SQRT_EIG = HBAR * 1e10 / math.sqrt(E_CHARGE * AMU)
INVCM = 100.0 * C_LIGHT * HPLANCK / E_CHARGE
RIGID_TOL = 1e-6


def rigid_basis(R, masses, periodic=False):
    """Orthonormal rigid basis (k, 3N) in mass-weighted coordinates: translations, then (free molecules) rotations about
    the centre of mass, two Gram-Schmidt passes in the order tx, ty, tz, rx, ry, rz; a vector keeping less than
    RIGID_TOL of its norm is dropped."""
    X = np.asarray(R, dtype=np.float64).reshape(-1, 3)
    m = np.asarray(masses, dtype=np.float64)
    sm = np.sqrt(m)
    d = X - (m[:, None] * X).sum(0) / m.sum()
    raw = []
    for a in range(3):
        v = np.zeros_like(X)
        v[:, a] = sm
        raw.append(v.ravel())
    if not periodic:
        for a in range(3):
            e = np.zeros(3)
            e[a] = 1.0
            raw.append((np.cross(e, d) * sm[:, None]).ravel())
    kept = []
    for v in raw:
        n0 = np.linalg.norm(v)
        v = v.copy()
        for _ in range(2):
            for u in kept:
                v -= (u @ v) * u
        n1 = np.linalg.norm(v)
        if n0 > 0 and n1 > RIGID_TOL * n0:
            kept.append(v / n1)
    return np.array(kept).reshape(-1, X.size)


def mass_weighted(H, masses):
    s = np.repeat(np.asarray(masses, dtype=np.float64) ** -0.5, 3)
    return 0.5 * (H + H.T) * np.outer(s, s)


def project(H, R, masses, periodic=False):
    """(Hp, n_rigid): Hp = P Hm P + c B^T B with P = I - B^T B and c = 2 |Hm|_inf + 1."""
    Hm = mass_weighted(np.asarray(H, dtype=np.float64), masses)
    B = rigid_basis(R, masses, periodic)
    P = np.eye(Hm.shape[0]) - B.T @ B
    c = 2.0 * np.abs(Hm).sum(1).max() + 1.0
    return P @ Hm @ P + c * (B.T @ B), B.shape[0]


def analyse(H, R, masses, periodic=False):
    """Eigenvalues of the vibrations (ascending, eV / (Angstrom^2 amu)), energies (eV, imaginary as negative),
    frequencies (cm^-1), Cartesian modes (n_vib, N, 3) as ASE's get_mode, and n_rigid, for H in eV / Angstrom^2."""
    Hp, k = project(H, R, masses, periodic)
    w, V = np.linalg.eigh(Hp)
    nv = Hp.shape[0] - k
    w, V = w[:nv], V[:, :nv]
    e = np.sign(w) * np.sqrt(np.abs(w)) * EV_PER_SQRT_EIG
    s = np.repeat(np.asarray(masses, dtype=np.float64) ** -0.5, 3)
    return {'eig': w, 'energies': e, 'frequencies': e / INVCM, 'modes': (V.T * s).reshape(nv, -1, 3), 'n_rigid': k}


def thermo(energies, T):
    """(ZPE, U_vib, S_vib, F_vib) of the positive energies (eV) at T (K), as ASE's HarmonicThermo."""
    e = np.asarray([x for x in energies if x > 0], dtype=np.float64)
    zpe = 0.5 * e.sum()
    if T == 0:
        return zpe, zpe, 0.0, zpe
    kT = KB_EV * T
    with np.errstate(over='ignore'):  # exp(e / kT) = inf at T -> 0: the thermal terms are 0
        U = zpe + (e / (np.exp(e / kT) - 1.0)).sum()
        S = KB_EV * ((e / kT) / (np.exp(e / kT) - 1.0) - np.log(1.0 - np.exp(-e / kT))).sum()
    return zpe, U, S, U - T * S


def vineyard(e_min, e_sad, E_min, E_sad, T):
    """(rate s^-1, prefactor s^-1): prod nu_min / prod nu_saddle(real) exp(-(E_sad - E_min) / kT), nu = e / h."""
    nu_min = np.asarray(e_min) * E_CHARGE / HPLANCK
    nu_sad = np.asarray([x for x in e_sad if x > 0]) * E_CHARGE / HPLANCK
    pref = math.exp(np.log(nu_min).sum() - np.log(nu_sad).sum())
    return pref * math.exp(-(E_sad - E_min) / (KB_EV * T)), pref
