"""Harmonic vibrational analysis of a model's stationary points on the device.

``GDMLVibrations(model, masses).analyse(positions)`` takes the Hessians of many geometries from
``GDMLPredict.predict_hessian``, mass-weights them and moves the rigid modes out of the way
(``sgdml_b200_vib_project``), then diagonalises them all at once (``sgdml_b200_symeig_batched``, one CTA per matrix, up
to ``sgdml_b200_symeig_max_n()`` coordinates; ``torch.linalg.eigh`` on the same device matrices above that).
``thermo`` gives harmonic vibrational thermochemistry as ASE's ``HarmonicThermo``, ``harmonic_rate`` the classical
harmonic transition-state-theory (Vineyard) rate between a minimum and a first-order saddle.

Units follow ASE and ``md.py``: positions in Angstrom, masses in amu, energies in eV, frequencies in cm^-1, temperature
in K, CODATA 2014 constants.  ``E_to_eV`` and ``F_to_eV_Ang`` convert the model's units as in ``GDMLDynamics``.
"""

import math

import numpy as np

from . import _lib
from .intf.ase_calc import _KCAL_PER_MOL_IN_EV
from .md import _AMU, _E_CHARGE, _HBAR, KB_EV
from .predict import GDMLPredict

_HPLANCK = 6.626070040e-34  # J s, CODATA 2014
_C = 299792458.0  # m / s
# hbar omega in eV from an eigenvalue of the mass-weighted Hessian in eV / (Angstrom^2 amu) (ASE's VibrationsData)
EV_PER_SQRT_EIG = _HBAR * 1e10 / math.sqrt(_E_CHARGE * _AMU)
INVCM = 100.0 * _C * _HPLANCK / _E_CHARGE  # eV per cm^-1 (ase.units.invcm)
H_EV_S = _HPLANCK / _E_CHARGE  # Planck's constant in eV s: nu = energy / H_EV_S


def symeig(A):
    """Eigenvalues (ascending) and eigenvectors (columns) of a stack of symmetric float64 CUDA matrices (B, n, n): the
    device Jacobi solver up to ``sgdml_b200_symeig_max_n()``, ``torch.linalg.eigh`` above it."""
    import torch

    B, n = A.shape[0], A.shape[-1]
    if n > _lib.lib().sgdml_b200_symeig_max_n():
        return torch.linalg.eigh(A)
    A = A.contiguous()
    w = torch.empty((B, n), dtype=torch.float64, device=A.device)
    V = torch.empty((B, n, n), dtype=torch.float64, device=A.device)
    _lib.check(_lib.lib().sgdml_b200_symeig_batched(_lib.ptr(A), n, B, _lib.ptr(w), _lib.ptr(V), _lib.current_stream()),
               'symeig_batched')
    return w, V


class GDMLVibrations(object):
    """Normal modes of a model at many geometries.

    model: a model dict or .npz path, or a ``GDMLPredict``.  masses: (N,) in amu.  A model with a cell is periodic: its
    rigid modes are the 3 translations only.

    The transition-state workflow: a saddle (``GDMLNEB``, ``GDMLDimer``) -> ``analyse(saddle)`` (exactly one imaginary
    mode) -> ``GDMLIRC(model, masses).run(saddle, modes[:, 0])`` -> the two minima it connects -> ``harmonic_rate`` from
    each of them over the saddle."""

    def __init__(self, model, masses, E_to_eV=_KCAL_PER_MOL_IN_EV, F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        import torch

        _lib.require_gpu()
        self.gdml_predict = model if isinstance(model, GDMLPredict) else GDMLPredict(
            model if isinstance(model, dict) else np.load(model, allow_pickle=True))
        self.n_atoms = self.gdml_predict.n_atoms
        self.E_to_eV = float(E_to_eV)
        self.F_to_eV_Ang = float(F_to_eV_Ang)
        self.Ang_to_R = self.F_to_eV_Ang / self.E_to_eV
        self.periodic = self.gdml_predict.lat_and_inv is not None
        masses = np.asarray(masses, dtype=np.float64).ravel()
        if masses.shape != (self.n_atoms,) or not np.all(masses > 0) or not np.all(np.isfinite(masses)):
            raise ValueError('masses must hold one positive value (amu) per atom: %d' % self.n_atoms)
        self.masses = masses
        self._ism = torch.from_numpy(masses ** -0.5).cuda()

    def analyse(self, positions):
        """positions (N, 3) or (B, N, 3) in Angstrom, a NumPy array or a float64 CUDA tensor.  Returns a dict of the
        same kind (geometry axis always present):
          frequencies (B, 3N) cm^-1: the vibrations ascending, imaginary ones as negative numbers, then n_rigid NaN
          energies (B, 3N) eV: hbar omega in the same layout;  modes (B, 3N, N, 3): the Cartesian displacement of each
          mode, the mass-weighted unit eigenvector times m^-1/2 (ASE's get_mode), NaN in the rigid slots
          n_rigid, n_imaginary (B,) int64;  zpe (B,) eV over the real modes;  hessian (B, 3N, 3N) eV / Angstrom^2 as
          predict_hessian returns it;  potential_energy (B,) eV;  fmax (B,) eV / Angstrom, the largest force on an
          atom (away from a stationary point the rigid modes carry curvature of order |F| |r|, and so do the others)."""
        import torch

        as_numpy = not hasattr(positions, 'data_ptr')
        if as_numpy:
            X = torch.from_numpy(np.ascontiguousarray(positions, dtype=np.float64)).cuda()
        else:
            if positions.dtype != torch.float64 or not positions.is_cuda:
                raise ValueError('positions: torch inputs must be float64 CUDA tensors')
            X = positions.contiguous()
        N, n = self.n_atoms, 3 * self.n_atoms
        if X.numel() % n != 0 or X.shape[-2:] != (N, 3) or X.dim() not in (2, 3):
            raise ValueError('positions must be (N, 3) or (B, N, 3) with N = %d' % N)
        X = X.reshape(-1, n)
        B = X.shape[0]
        gp = self.gdml_predict
        R = (X * self.Ang_to_R).contiguous()
        E, F = gp.predict(R)
        H = gp.predict_hessian(R) * (self.E_to_eV * self.Ang_to_R ** 2)
        Hp = torch.empty_like(H)
        n_rigid = torch.empty(B, dtype=torch.int64, device=H.device)
        if B > 0:
            _lib.check(_lib.lib().sgdml_b200_vib_project(
                _lib.ptr(H), _lib.ptr(X), _lib.ptr(self._ism), B, N, int(self.periodic), _lib.ptr(Hp),
                _lib.ptr(n_rigid), _lib.current_stream()), 'vib_project')
        w, V = symeig(Hp) if B > 0 else (torch.empty((0, n), dtype=torch.float64, device=H.device), Hp)
        vib = torch.arange(n, device=H.device)[None, :] < (n - n_rigid)[:, None]
        nan = torch.tensor(float('nan'), dtype=torch.float64, device=H.device)
        energies = torch.where(vib, torch.sign(w) * torch.sqrt(torch.abs(w)) * EV_PER_SQRT_EIG, nan)
        modes = V.transpose(1, 2) * self._ism.repeat_interleave(3)[None, None, :]
        modes = torch.where(vib[:, :, None], modes, nan).reshape(B, n, N, 3)
        f = (F * self.F_to_eV_Ang).reshape(B, N, 3)
        out = {
            'frequencies': energies / INVCM,
            'energies': energies,
            'modes': modes,
            'n_rigid': n_rigid,
            'n_imaginary': (vib & (w < 0)).sum(1),
            'zpe': 0.5 * torch.where(vib & (w > 0), energies, torch.zeros_like(energies)).sum(1),
            'hessian': H,
            'potential_energy': E * self.E_to_eV,
            'fmax': torch.sqrt((f * f).sum(-1)).amax(-1) if N > 0 and B > 0 else torch.zeros(B, dtype=torch.float64),
        }
        return {k: v.cpu().numpy() for k, v in out.items()} if as_numpy else out


def _host(x):
    return x.detach().cpu().numpy() if hasattr(x, 'data_ptr') else np.asarray(x)


def _vib_energies(result):
    """(B, 3N) eV of the vibrations (NaN in the rigid slots) and (B,) counts of imaginary modes, on the host."""
    return _host(result['energies']).astype(np.float64), _host(result['n_imaginary']).astype(np.int64)


def thermo(result, temperature_K):
    """Harmonic vibrational thermochemistry of each geometry of an ``analyse`` result at `temperature_K`, as ASE's
    HarmonicThermo over the real modes (imaginary ones excluded and counted):
      U_vib = ZPE + sum e / (exp(e / kT) - 1),  S_vib = k sum [(e / kT) / (exp(e / kT) - 1) - ln(1 - exp(-e / kT))],
      F_vib = U_vib - T S_vib.
    Returns {'zpe', 'U_vib', 'F_vib'} in eV, {'S_vib'} in eV / K, 'n_excluded' (the imaginary modes), each (B,)."""
    T = float(temperature_K)
    if not T >= 0.0 or not math.isfinite(T):
        raise ValueError('temperature_K must be finite and >= 0')
    e, n_imag = _vib_energies(result)
    real = np.isfinite(e) & (e > 0)
    e = np.where(real, e, 1.0)
    zpe = 0.5 * np.where(real, e, 0.0).sum(-1)
    if T == 0.0:
        zero = np.zeros_like(zpe)
        return {'zpe': zpe, 'U_vib': zpe.copy(), 'S_vib': zero, 'F_vib': zpe.copy(), 'n_excluded': n_imag}
    kT = KB_EV * T
    x = e / kT
    with np.errstate(over='ignore'):  # expm1(x) = inf for e >> kT: that mode's thermal terms are 0
        em1 = np.expm1(x)
    U = zpe + np.where(real, e / em1, 0.0).sum(-1)
    S = KB_EV * np.where(real, x / em1 - np.log(-np.expm1(-x)), 0.0).sum(-1)
    return {'zpe': zpe, 'U_vib': U, 'S_vib': S, 'F_vib': U - T * S, 'n_excluded': n_imag}


def harmonic_rate(minimum, saddle, temperature_K):
    """Classical harmonic transition-state-theory (Vineyard) rate from a minimum over a first-order saddle, per geometry
    pair of two ``analyse`` results (B each, or one of them B = 1):
      k = (prod_i nu_i^min / prod_j nu_j^saddle) exp(-(E_saddle - E_min) / kT),
    nu = hbar omega / h over the vibrations (the saddle's real ones), evaluated in log space.  Returns {'rate'} in s^-1,
    {'prefactor'} in s^-1, {'barrier'} in eV and {'log_rate'}.  Raises ValueError unless every minimum has no imaginary
    mode, every saddle exactly one, and both have the same number of rigid modes.  Which minimum a saddle leads to is
    the caller's claim; ``GDMLIRC.run(saddle, analyse(saddle)['modes'][:, 0])`` finds the two minima it connects, one
    rate per direction."""
    T = float(temperature_K)
    if not T > 0.0 or not math.isfinite(T):
        raise ValueError('temperature_K must be finite and > 0')
    e_min, i_min = _vib_energies(minimum)
    e_sad, i_sad = _vib_energies(saddle)
    r_min, r_sad = _host(minimum['n_rigid']), _host(saddle['n_rigid'])
    if np.any(i_min != 0):
        raise ValueError('the minimum has imaginary modes: %s' % i_min)
    if np.any(i_sad != 1):
        raise ValueError('the saddle must have exactly one imaginary mode: %s' % i_sad)
    if np.any(np.broadcast_to(r_min, np.broadcast(r_min, r_sad).shape) != r_sad):
        raise ValueError('the minimum and the saddle have different rigid-mode counts: %s, %s' % (r_min, r_sad))
    vm, vs = np.isfinite(e_min), np.isfinite(e_sad) & (e_sad > 0)
    if np.any(np.where(vm, e_min, 1.0) <= 0.0):
        raise ValueError('the minimum has a zero-frequency vibration')
    log_nu_min = np.where(vm, np.log(np.where(vm, e_min, 1.0) / H_EV_S), 0.0).sum(-1)
    log_nu_sad = np.where(vs, np.log(np.where(vs, e_sad, 1.0) / H_EV_S), 0.0).sum(-1)
    log_pref = log_nu_min - log_nu_sad
    barrier = _host(saddle['potential_energy']) - _host(minimum['potential_energy'])
    log_rate = log_pref - barrier / (KB_EV * T)
    return {'rate': np.exp(log_rate), 'prefactor': np.exp(log_pref), 'barrier': barrier, 'log_rate': log_rate}
