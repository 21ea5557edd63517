"""``GDMLDynamics`` -- molecular dynamics of many replicas on the device (``sgdml_b200_md_*`` in
include/sgdml_b200.h): velocity-Verlet (NVE) and BAOAB Langevin (NVT) trajectories, many steps per call, with
positions, velocities and forces kept in GPU memory between steps.  ``GDMLPathIntegralDynamics`` -- path-integral MD
of ring polymers on the same engine (``sgdml_b200_pimd_*``): PILE-L thermostatted (or NVE) ring-polymer trajectories
with the primitive and centroid-virial quantum kinetic-energy estimators.

``GDMLReplicaExchange`` -- temperature replica exchange (parallel tempering) on the same engine
(``sgdml_b200_remd_run``): ladders of Langevin replicas at fixed temperatures whose neighbours swap configurations by a
Metropolis test inside the step graph.

``GDMLNPTDynamics`` -- constant-pressure MD of periodic models on the same engine (``sgdml_b200_npt_*``): Langevin
replicas, each in a cell of its own that an isotropic stochastic cell rescaling barostat scales.

``GDMLMetadynamics`` -- well-tempered multiple-walker metadynamics on the same engine (``sgdml_b200_metad_*``):
groups of Langevin walkers, each group sharing one store of Gaussian hills on distance, angle and dihedral collective
variables, for free-energy surfaces along chosen coordinates.  ``GDMLUmbrellaSampling`` -- umbrella sampling on the
same CVs with replica exchange between neighbouring windows (``sgdml_b200_umbrella_*``), unbiased by MBAR on the device.

``GDMLRelaxation`` -- geometry optimisation of many replicas on the same engine (``sgdml_b200_relax_*``): FIRE and
L-BFGS, each replica frozen once it has converged.  ``GDMLNEB`` and ``GDMLDimer`` find saddle points on it: between
two minima with the nudged elastic band (``sgdml_b200_neb_fire``), or next to one minimum with the dimer method
(``sgdml_b200_dimer_fire``).  ``GDMLIRC`` follows the intrinsic reaction coordinate down from a saddle to the two minima
it connects (``sgdml_b200_irc_rk4``).

Units follow ASE and ``intf.ase_calc.SGDMLCalculator``: positions in Angstrom, velocities in Angstrom/fs, masses in
amu, energies in eV, time in fs, temperature in K.  ``E_to_eV`` and ``F_to_eV_Ang`` convert the model's units as in
the calculator (defaults: kcal/mol and Angstrom).  Internally the engine works in the model's units with the
femtosecond as its time unit.
"""

import ctypes
import math

import numpy as np

from . import _lib
from .intf.ase_calc import _KCAL_PER_MOL_IN_EV
from .predict import GDMLPredict

# CODATA 2014, the values ASE's units use by default (and that _KCAL_PER_MOL_IN_EV is built from)
_E_CHARGE = 1.6021766208e-19  # C
_AMU = 1.660539040e-27  # kg
_K_B = 1.38064852e-23  # J / K
FS = 1e-15 * 1e10 * np.sqrt(_E_CHARGE / _AMU)  # ase.units.fs: 1 fs in ASE's time unit Angstrom sqrt(amu / eV)
KB_EV = _K_B / _E_CHARGE  # ase.units.kB: eV / K
_HBAR = 1.054571800e-34  # J s
HBAR_EV_FS = _HBAR / _E_CHARGE * 1e15  # eV fs (0.6582119514)


class GDMLDynamics(object):
    """Trajectories of `n_replicas` copies of one model's system.

    model: a model dict or .npz path (as ``SGDMLCalculator``), or a ``GDMLPredict``.  masses: (N,) in amu (e.g.
    ``atoms.get_masses()``; the model stores atomic numbers, the engine has no element table).

    ``set_state(positions, velocities=None, step=0)`` starts (or restarts) every replica: positions (n_replicas, N, 3)
    [or (N, 3) for one replica] in Angstrom, velocities in Angstrom/fs (None: at rest), `step` the step index the
    random stream continues from.  NumPy arrays or float64 CUDA tensors; ``run`` and ``get_state`` return the same
    kind.  ``run(n_steps, dt_fs, temperature_K=0, friction_per_fs=0, seed=0, stride=0)`` integrates and returns the
    frames after every `stride`-th step: {'positions', 'velocities': (n_frames, n_replicas, N, 3), 'potential_energy',
    'kinetic_energy': (n_frames, n_replicas)} in Angstrom, Angstrom/fs and eV (stride 0: an empty dict).  Zero friction
    is velocity Verlet; a temperature needs friction.

    The model's F and E stored by ``set_state`` are not refreshed if the model changes afterwards: call ``set_state``
    again then."""

    def __init__(self, model, masses, n_replicas=1, E_to_eV=_KCAL_PER_MOL_IN_EV, F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self._init_model(model, n_replicas, E_to_eV, F_to_eV_Ang)
        masses = np.ascontiguousarray(np.asarray(masses, dtype=np.float64).ravel())
        if masses.shape != (self.n_atoms,):
            raise ValueError('masses must hold one value (amu) per atom: %d' % self.n_atoms)
        # a = F inv_mass in model length per fs^2, F in the model's force unit
        self.inv_mass = self.F_to_eV_Ang * self.Ang_to_R * FS**2 / masses
        self._handle = self._create_handle()

    def _init_model(self, model, n_replicas, E_to_eV, F_to_eV_Ang):
        _lib.require_gpu()
        self.gdml_predict = model if isinstance(model, GDMLPredict) else GDMLPredict(
            model if isinstance(model, dict) else np.load(model, allow_pickle=True))
        self.n_atoms = self.gdml_predict.n_atoms
        self.n_replicas = int(n_replicas)
        self.E_to_eV = float(E_to_eV)
        self.F_to_eV_Ang = float(F_to_eV_Ang)
        self.Ang_to_R = self.F_to_eV_Ang / self.E_to_eV  # Angstrom -> model length unit (ase_calc.py:93-94)
        self._torch_device = None

    def _create_handle(self):
        handle = ctypes.c_void_p()
        _lib.check(
            _lib.lib().sgdml_b200_md_create(ctypes.byref(handle), self.gdml_predict._handle, self.n_replicas,
                                            _lib.ptr(self.inv_mass)),
            'md_create',
        )
        return handle

    def __del__(self):
        h = getattr(self, '_handle', None)
        if h is not None and h.value:
            try:
                _lib.lib().sgdml_b200_md_destroy(h)
            except Exception:
                pass
            self._handle = None

    # ------------------------------------------------------------------ arrays
    def _flat(self, x, name):
        dimi = 3 * self.n_atoms
        if hasattr(x, 'data_ptr'):
            import torch

            if x.dtype != torch.float64 or not x.is_cuda:
                raise ValueError('%s: torch inputs must be float64 CUDA tensors' % name)
            n = x.numel()
        else:
            x = np.ascontiguousarray(x, dtype=np.float64)
            n = x.size
        if n != self.n_replicas * dimi:
            raise ValueError('%s must hold n_replicas x 3N = %d x %d values' % (name, self.n_replicas, dimi))
        return x.reshape(self.n_replicas, dimi).contiguous() if hasattr(x, 'data_ptr') else x.reshape(self.n_replicas, dimi)

    @property
    def _shape(self):
        """The shape ``get_state`` and ``run`` give the replica axis."""
        return (self.n_replicas,)

    def _empty(self, shape, dtype=np.float64):
        if self._torch_device is None:
            return np.empty(shape, dtype=dtype)
        import torch

        return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), device=self._torch_device)

    # ------------------------------------------------------------------ model units (L, model energy, fs)
    def _set_state_raw(self, R, V=None, step=0):
        R = self._flat(R, 'positions')
        V = None if V is None else self._flat(V, 'velocities')
        if V is not None and hasattr(V, 'data_ptr') != hasattr(R, 'data_ptr'):
            raise ValueError('positions and velocities must be of the same kind')
        _lib.check(
            _lib.lib().sgdml_b200_md_set_state(self._handle, _lib.ptr(R), _lib.ptr(V), int(step), _lib.current_stream()),
            'md_set_state',
        )
        self._torch_device = R.device if hasattr(R, 'data_ptr') else None

    def _get_state_raw(self):
        shape = (self.n_replicas, 3 * self.n_atoms)
        R, V, F, E = self._empty(shape), self._empty(shape), self._empty(shape), self._empty((self.n_replicas,))
        step = np.zeros(1, dtype=np.uint64)
        _lib.check(
            _lib.lib().sgdml_b200_md_get_state(self._handle, _lib.ptr(R), _lib.ptr(V), _lib.ptr(F), _lib.ptr(E),
                                               _lib.ptr(step), _lib.current_stream()),
            'md_get_state',
        )
        return {'R': R, 'V': V, 'F': F, 'E_pot': E, 'step': int(step[0])}

    def _frames(self, n_steps, stride, frames, n_poly=0):
        """Empty frame arrays for the names in `frames`: (n_frames, n_replicas, 3N) for R and V, (n_frames, n_replicas, 9)
        for the NPT cells, (n_frames, n_poly) for K_prim and K_cv, else (n_frames, n_replicas), int32 for the walker
        labels; {} when the run writes no frames."""
        n_frames = n_steps // stride if stride > 0 and n_steps % stride == 0 else 0
        dims = {'R': (self.n_replicas, 3 * self.n_atoms), 'V': (self.n_replicas, 3 * self.n_atoms), 'K_prim': (n_poly,),
                'K_cv': (n_poly,), 'cell': (self.n_replicas, 9)}
        return {k: self._empty((n_frames,) + dims.get(k, (self.n_replicas,)), np.int32 if k == 'walker' else np.float64)
                for k in frames} if n_frames > 0 else {}

    def _run_raw(self, n_steps, dt, gamma=0.0, kT=0.0, seed=0, stride=0, frames=('R', 'V', 'E_pot', 'E_kin')):
        n_steps, stride = int(n_steps), int(stride)
        out = self._frames(n_steps, stride, frames)
        _lib.check(
            _lib.lib().sgdml_b200_md_run(self._handle, n_steps, float(dt), float(gamma), float(kT), int(seed), stride,
                                         *(_lib.ptr(out.get(k)) for k in ('R', 'V', 'E_pot', 'E_kin')),
                                         _lib.current_stream()),
            'md_run',
        )
        return out

    # ------------------------------------------------------------------ ASE units
    def set_state(self, positions, velocities=None, step=0):
        R = self._flat(positions, 'positions') * self.Ang_to_R
        V = None if velocities is None else self._flat(velocities, 'velocities') * self.Ang_to_R
        self._set_state_raw(R, V, step)

    def get_state(self):
        """{'positions', 'velocities', 'forces' (n_replicas, N, 3), 'potential_energy' (n_replicas,), 'step'}: Angstrom,
        Angstrom/fs, eV/Angstrom, eV.  Path-integral and replica-exchange handles shape the replica axis (n_polymers,
        n_beads) and (n_ladders, n_temps)."""
        s = self._get_state_raw()
        g, a = self._shape, (self.n_atoms, 3)
        return {'positions': (s['R'] / self.Ang_to_R).reshape(g + a),
                'velocities': (s['V'] / self.Ang_to_R).reshape(g + a),
                'forces': (s['F'] * self.F_to_eV_Ang).reshape(g + a),
                'potential_energy': (s['E_pot'] * self.E_to_eV).reshape(g), 'step': s['step']}

    def _ase_frames(self, f):
        """The frames R, V, E_pot, E_kin among f (model units) in ASE units, shaped (n_frames,) + _shape [+ (N, 3)]."""
        out = {}
        for k, name in (('R', 'positions'), ('V', 'velocities')):
            if k in f:
                out[name] = (f[k] / self.Ang_to_R).reshape((f[k].shape[0],) + self._shape + (self.n_atoms, 3))
        for k, name in (('E_pot', 'potential_energy'), ('E_kin', 'kinetic_energy')):
            if k in f:
                out[name] = (f[k] * self.E_to_eV).reshape((f[k].shape[0],) + self._shape)
        return out

    def run(self, n_steps, dt_fs, temperature_K=0.0, friction_per_fs=0.0, seed=0, stride=0):
        kT = KB_EV * float(temperature_K) / self.E_to_eV
        return self._ase_frames(self._run_raw(n_steps, dt_fs, friction_per_fs, kT, seed, stride))


class GDMLPathIntegralDynamics(GDMLDynamics):
    """Path-integral MD of `n_polymers` ring polymers of `n_beads` beads (1 to 64) each, in the units of
    ``GDMLDynamics``.  Bead j of polymer p is replica p n_beads + j of the engine's handle.

    ``set_state(positions, velocities=None, step=0)``: positions (n_polymers, n_beads, N, 3), or (n_polymers, N, 3) /
    (N, 3) copied to every bead (and polymer); velocities likewise (None: at rest).
    ``run(n_steps, dt_fs, temperature_K, centroid_friction_per_fs=0, pile_lambda=1, seed=0, stride=0)`` integrates
    with the PILE-L thermostat (the centroid mode at the given friction, internal mode k at 2 pile_lambda omega_k:
    pile_lambda = 1 damps every internal mode critically, 0.5 with zero centroid friction is thermostatted RPMD, zero
    for both is NVE RPMD) and returns the frames after every `stride`-th step: {'positions', 'velocities':
    (n_frames, n_polymers, n_beads, N, 3), 'potential_energy': (n_frames, n_polymers, n_beads),
    'kinetic_energy_primitive', 'kinetic_energy_virial': (n_frames, n_polymers)} in Angstrom, Angstrom/fs and eV (the
    kinetic energies are the quantum estimators of the whole molecule; stride 0: an empty dict).  A ring polymer
    needs a temperature > 0; with one bead ``run`` is ``GDMLDynamics.run`` bit for bit."""

    def __init__(self, model, masses, n_beads, n_polymers=1, E_to_eV=_KCAL_PER_MOL_IN_EV,
                 F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.n_beads = int(n_beads)
        self.n_polymers = int(n_polymers)
        super().__init__(model, masses, self.n_polymers * self.n_beads, E_to_eV, F_to_eV_Ang)

    def _create_handle(self):
        handle = ctypes.c_void_p()
        _lib.check(
            _lib.lib().sgdml_b200_pimd_create(ctypes.byref(handle), self.gdml_predict._handle, self.n_polymers,
                                              self.n_beads, _lib.ptr(self.inv_mass)),
            'pimd_create',
        )
        return handle

    @property
    def _shape(self):
        return (self.n_polymers, self.n_beads)

    def _beads(self, x, name):
        """(n_polymers, n_beads, N, 3), (n_polymers, N, 3) or (N, 3) -> (n_polymers n_beads, 3N)."""
        return _groups(x, name, self.n_polymers, self.n_beads, self.n_atoms, ('n_polymers', 'n_beads'))

    # ------------------------------------------------------------------ model units (L, model energy, fs)
    def _run_raw(self, n_steps, dt, kT, hbar, gamma=0.0, lam=0.0, seed=0, stride=0,
                 frames=('R', 'V', 'E_pot', 'E_kin', 'K_prim', 'K_cv')):
        n_steps, stride = int(n_steps), int(stride)
        out = self._frames(n_steps, stride, frames, self.n_polymers)
        _lib.check(
            _lib.lib().sgdml_b200_pimd_run(self._handle, n_steps, float(dt), float(kT), float(hbar), float(gamma),
                                           float(lam), int(seed), stride,
                                           *(_lib.ptr(out.get(k)) for k in ('R', 'V', 'E_pot', 'E_kin', 'K_prim',
                                                                           'K_cv')),
                                           _lib.current_stream()),
            'pimd_run',
        )
        return out

    # ------------------------------------------------------------------ ASE units
    def set_state(self, positions, velocities=None, step=0):
        positions = self._beads(positions, 'positions')
        velocities = None if velocities is None else self._beads(velocities, 'velocities')
        super().set_state(positions, velocities, step)

    def run(self, n_steps, dt_fs, temperature_K, centroid_friction_per_fs=0.0, pile_lambda=1.0, seed=0, stride=0):
        kT = KB_EV * float(temperature_K) / self.E_to_eV
        hbar = HBAR_EV_FS / self.E_to_eV
        f = self._run_raw(n_steps, dt_fs, kT, hbar, centroid_friction_per_fs, pile_lambda, seed, stride,
                          frames=('R', 'V', 'E_pot', 'K_prim', 'K_cv'))
        if not f:
            return {}
        out = self._ase_frames(f)
        out.update(kinetic_energy_primitive=f['K_prim'] * self.E_to_eV, kinetic_energy_virial=f['K_cv'] * self.E_to_eV)
        return out


def _groups(x, name, n_g, per, N, axes):
    """(n_g, per, N, 3), (n_g, N, 3) or (N, 3), the last two copied to every member (and group), as (n_g, per, N, 3);
    axes names n_g and per in the error message."""
    shape = tuple(x.shape)
    if shape == (n_g, per, N, 3):
        return x
    if shape == (n_g, N, 3) or shape == (N, 3):
        x = x.reshape(-1, 1, N, 3)
        if hasattr(x, 'data_ptr'):
            return x.expand(n_g, per, N, 3).contiguous()
        return np.ascontiguousarray(np.broadcast_to(np.asarray(x, dtype=np.float64), (n_g, per, N, 3)))
    raise ValueError('%s must be (%s, %s, N, 3), (%s, N, 3) or (N, 3) = (%d, %d, %d, 3): %s'
                     % ((name,) + axes + axes[:1] + (n_g, per, N, shape)))


class GDMLReplicaExchange(GDMLDynamics):
    """Temperature replica exchange (parallel tempering; Sugita & Okamoto, Chem. Phys. Lett. 314, 141 (1999)) of
    `n_ladders` ladders of Langevin replicas, in the units of ``GDMLDynamics``.  Slot k of ladder l (replica
    l n_temps + k of the engine's handle) stays at temperatures_K[k] for the whole run; neighbours in `temperatures_K`
    swap configurations by the Metropolis test, with the velocities rescaled to the new temperature, so every output is
    sorted by temperature.  A geometric ladder, ``np.geomspace(T_low, T_high, n_temps)``, gives neighbours about equal
    acceptance when the heat capacity varies little.  The exchanges run inside the step graph on the energies already in
    device memory: no host round trip per exchange.  A walker label follows each configuration: the slot it held at
    ``set_state``.

    ``set_state(positions, velocities=None, step=0)``: positions (n_ladders, n_temps, N, 3), or (n_ladders, N, 3) /
    (N, 3) copied to every slot (and ladder); velocities likewise (None: at rest).  ``set_state`` resets the walker
    labels to the slots.  ``get_state()`` as ``GDMLDynamics``'s, shaped (n_ladders, n_temps, ...).
    ``run(n_steps, dt_fs, friction_per_fs, exchange_every, seed=0, stride=0)`` integrates every slot with BAOAB
    Langevin at its temperature (friction > 0) and attempts exchanges on every `exchange_every`-th state, alternating
    the even and odd neighbour pairs (0: no exchanges).  It returns {'positions', 'velocities': (n_frames, n_ladders,
    n_temps, N, 3), 'potential_energy', 'kinetic_energy', 'walker': (n_frames, n_ladders, n_temps)} after every
    `stride`-th step (none for stride 0), and always 'walkers' (n_ladders, n_temps), the labels after the run, and
    'n_accepted', 'n_attempted' (int64) and 'acceptance' (their ratio, NaN without attempts), (n_ladders, n_temps - 1),
    this run's swaps of each neighbour pair (k, k + 1).  Angstrom, Angstrom/fs and eV; NumPy arrays or float64 CUDA
    tensors in, the same kind out.  A run continued over several calls is one long run."""

    def __init__(self, model, masses, temperatures_K, n_ladders=1, E_to_eV=_KCAL_PER_MOL_IN_EV,
                 F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.temperatures_K = np.array(temperatures_K, dtype=np.float64).ravel()
        self.n_temps = len(self.temperatures_K)
        self.n_ladders = int(n_ladders)
        if self.n_temps < 2 or self.n_ladders < 1:
            raise ValueError('a ladder needs at least two temperatures, and n_ladders >= 1')
        super().__init__(model, masses, self.n_ladders * self.n_temps, E_to_eV, F_to_eV_Ang)

    @property
    def _shape(self):
        return (self.n_ladders, self.n_temps)

    # ------------------------------------------------------------------ model units (L, model energy, fs)
    def _run_raw(self, n_steps, dt, gamma, kT, exchange_every, seed=0, stride=0,
                 frames=('R', 'V', 'E_pot', 'E_kin', 'walker')):
        """kT (n_temps,) in the model's energy unit.  -> frames and 'walkers' (n_replicas,), 'n_accepted',
        'n_attempted' (n_ladders, n_temps - 1)."""
        n_steps, stride = int(n_steps), int(stride)
        out = self._frames(n_steps, stride, frames)
        kT = np.ascontiguousarray(kT, dtype=np.float64)
        if kT.shape != (self.n_temps,):
            raise ValueError('kT must hold one value per temperature: %d' % self.n_temps)
        walkers = self._empty((self.n_replicas,), np.int32)
        acc, att = (self._empty((self.n_ladders, self.n_temps - 1), np.int64) for _ in range(2))
        _lib.check(
            _lib.lib().sgdml_b200_remd_run(self._handle, self.n_temps, _lib.ptr(kT), n_steps, float(dt), float(gamma),
                                           int(seed), int(exchange_every), stride,
                                           *(_lib.ptr(out.get(k)) for k in ('R', 'V', 'E_pot', 'E_kin', 'walker')),
                                           _lib.ptr(walkers), _lib.ptr(acc), _lib.ptr(att), _lib.current_stream()),
            'remd_run',
        )
        out.update(walkers=walkers, n_accepted=acc, n_attempted=att)
        return out

    # ------------------------------------------------------------------ ASE units
    def set_state(self, positions, velocities=None, step=0):
        axes = ('n_ladders', 'n_temps')
        positions = _groups(positions, 'positions', self.n_ladders, self.n_temps, self.n_atoms, axes)
        if velocities is not None:
            velocities = _groups(velocities, 'velocities', self.n_ladders, self.n_temps, self.n_atoms, axes)
        super().set_state(positions, velocities, step)

    def run(self, n_steps, dt_fs, friction_per_fs, exchange_every, seed=0, stride=0):
        kT = KB_EV * self.temperatures_K / self.E_to_eV
        f = self._run_raw(n_steps, dt_fs, friction_per_fs, kT, exchange_every, seed, stride)
        acc, att = f['n_accepted'], f['n_attempted']
        if hasattr(att, 'data_ptr'):
            ratio = acc.double() / att.clip(1).double()
        else:
            ratio = acc / att.clip(1)
        ratio[att == 0] = np.nan
        out = {'walkers': f['walkers'].reshape(self._shape), 'n_accepted': acc, 'n_attempted': att, 'acceptance': ratio}
        out.update(self._ase_frames(f))
        if 'walker' in f:
            out['walker'] = f['walker'].reshape((f['walker'].shape[0],) + self._shape)
        return out


class GDMLNPTDynamics(GDMLDynamics):
    """Constant-pressure (NPT) molecular dynamics of `n_replicas` replicas of a periodic model, in the units of
    ``GDMLDynamics``: BAOAB Langevin with the isotropic stochastic cell rescaling barostat of Bernetti & Bussi
    (J. Chem. Phys. 153, 114107 (2020)).  Every replica lives in a cell of its own, which the barostat scales with the
    positions; the step, the forces and the virial run on the device, with no host round trip per step.

    cells: (n_replicas, 3, 3) or (3, 3) in Angstrom with the lattice vectors as ROWS (ASE's ``atoms.cell``); None: the
    model's own cell for every replica (a free-molecule model has none and raises).  NumPy arrays or torch tensors.
    ``set_state(positions, velocities=None, step=0)`` as ``GDMLDynamics``'s; forces, energies and stresses are
    evaluated in each replica's cell.  ``set_cells(cells)`` replaces the cells (positions do not move).
    ``get_state()`` adds 'cells' (n_replicas, 3, 3) and 'stress' (n_replicas, 6), -W / V in eV/Angstrom^3 in Voigt
    order (xx, yy, zz, yz, xz, xy), the calculator's 'stress'.
    ``run(n_steps, dt_fs, temperature_K, friction_per_fs, pressure_au, compressibility_au, taup_fs, seed=0, stride=0)``
    integrates at the target pressure (eV/Angstrom^3) with the isothermal compressibility (Angstrom^3/eV) and barostat
    time constant taup_fs, the names and units of ASE's barostats; zero compressibility keeps every cell fixed.  It
    returns ``GDMLDynamics.run``'s frames plus 'cells' (n_frames, n_replicas, 3, 3), 'volume' (Angstrom^3) and
    'pressure' (eV/Angstrom^3, the instantaneous (2 E_kin + tr W) / 3V), (n_frames, n_replicas).  NumPy arrays or
    float64 CUDA tensors in, the same kind out.  Positions are never wrapped into the cell."""

    def __init__(self, model, masses, cells=None, n_replicas=1, E_to_eV=_KCAL_PER_MOL_IN_EV,
                 F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self._cells_arg = cells
        super().__init__(model, masses, n_replicas, E_to_eV, F_to_eV_Ang)

    def _raw_cells(self, cells):
        """cells in Angstrom (rows), or None -> (lattices, inverses) (n_replicas, 9) in model units (columns)."""
        n = self.n_replicas
        if cells is None:
            if self.gdml_predict.lat_and_inv is None:
                raise ValueError('a free-molecule model has no cell: pass cells (Angstrom, vectors as rows)')
            lat, inv = self.gdml_predict.lat_and_inv
            return (np.ascontiguousarray(np.broadcast_to(np.asarray(lat, dtype=np.float64).reshape(1, 9), (n, 9))),
                    np.ascontiguousarray(np.broadcast_to(np.asarray(inv, dtype=np.float64).reshape(1, 9), (n, 9))))
        c = cells.detach().cpu().numpy() if hasattr(cells, 'data_ptr') else cells
        c = np.asarray(c, dtype=np.float64)
        if c.shape == (3, 3):
            c = np.broadcast_to(c, (n, 3, 3))
        if c.shape != (n, 3, 3):
            raise ValueError('cells must be (n_replicas, 3, 3) or (3, 3) = (%d, 3, 3): %s' % (n, c.shape))
        lat = np.ascontiguousarray(c.swapaxes(-1, -2) * self.Ang_to_R)
        return lat.reshape(n, 9), np.ascontiguousarray(np.linalg.inv(lat)).reshape(n, 9)

    def _create_handle(self):
        lat, inv = self._raw_cells(self._cells_arg)
        handle = ctypes.c_void_p()
        _lib.check(
            _lib.lib().sgdml_b200_npt_create(ctypes.byref(handle), self.gdml_predict._handle, self.n_replicas,
                                             _lib.ptr(self.inv_mass), _lib.ptr(lat), _lib.ptr(inv)),
            'npt_create',
        )
        return handle

    # ------------------------------------------------------------------ model units (L, model energy, fs)
    def _set_cells_raw(self, lattices, lattice_invs):
        """(n_replicas, 9) HOST arrays each, model units, vectors as columns."""
        lat = np.ascontiguousarray(lattices, dtype=np.float64)
        inv = np.ascontiguousarray(lattice_invs, dtype=np.float64)
        if lat.size != 9 * self.n_replicas or inv.size != 9 * self.n_replicas:
            raise ValueError('lattices and lattice_invs must hold n_replicas x 9 values each: %d' % self.n_replicas)
        _lib.check(_lib.lib().sgdml_b200_npt_set_cells(self._handle, _lib.ptr(lat), _lib.ptr(inv),
                                                       _lib.current_stream()), 'npt_set_cells')

    def _get_cells_raw(self):
        """{'lattice', 'lattice_inv', 'W'}: (n_replicas, 9) each, model units."""
        out = {k: self._empty((self.n_replicas, 9)) for k in ('lattice', 'lattice_inv', 'W')}
        _lib.check(
            _lib.lib().sgdml_b200_npt_get_cells(self._handle, *(_lib.ptr(out[k]) for k in ('lattice', 'lattice_inv', 'W')),
                                                _lib.current_stream()),
            'npt_get_cells',
        )
        return out

    def _run_raw(self, n_steps, dt, gamma, kT, P0, beta_T, tau_p, seed=0, stride=0,
                 frames=('R', 'V', 'E_pot', 'E_kin', 'cell', 'P')):
        n_steps, stride = int(n_steps), int(stride)
        out = self._frames(n_steps, stride, frames)
        _lib.check(
            _lib.lib().sgdml_b200_npt_run(self._handle, n_steps, float(dt), float(gamma), float(kT), float(P0),
                                          float(beta_T), float(tau_p), int(seed), stride,
                                          *(_lib.ptr(out.get(k)) for k in ('R', 'V', 'E_pot', 'E_kin', 'cell', 'P')),
                                          _lib.current_stream()),
            'npt_run',
        )
        return out

    # ------------------------------------------------------------------ ASE units
    def _ase_cells(self, lat):
        """(..., 9) model-unit lattices (columns) -> (..., 3, 3) Angstrom cells (rows) and their volumes (...)."""
        c = lat.reshape(lat.shape[:-1] + (3, 3)).swapaxes(-1, -2) / self.Ang_to_R
        return c, abs(_det3(c))

    def set_cells(self, cells):
        self._set_cells_raw(*self._raw_cells(cells))

    def get_state(self):
        out = super().get_state()
        c = self._get_cells_raw()
        cells, vol = self._ase_cells(c['lattice'])
        s = -c['W'].reshape(-1, 3, 3) * self.E_to_eV / vol.reshape(-1, 1, 1)
        out.update(cells=cells, stress=s[:, [0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]])
        return out

    def run(self, n_steps, dt_fs, temperature_K, friction_per_fs, pressure_au, compressibility_au, taup_fs, seed=0,
            stride=0):
        kT = KB_EV * float(temperature_K) / self.E_to_eV
        vol_unit = self.Ang_to_R**3  # Angstrom^3 -> L^3
        f = self._run_raw(n_steps, dt_fs, friction_per_fs, kT, float(pressure_au) / (self.E_to_eV * vol_unit),
                          float(compressibility_au) * self.E_to_eV * vol_unit, taup_fs, seed, stride)
        out = self._ase_frames(f)
        if 'cell' in f:
            out['cells'], out['volume'] = self._ase_cells(f['cell'])
            out['pressure'] = f['P'] * (self.E_to_eV * vol_unit)
        return out


_CV_TYPES = {'distance': 0, 'angle': 1, 'dihedral': 2}


def _cv_list(cvs, what):
    """[(kind, atoms)] checked: 1 to 4 CVs of a known kind, each with its number of atoms"""
    cvs = list(cvs)
    if not 1 <= len(cvs) <= 4:
        raise ValueError('%s takes 1 to 4 collective variables: %d' % (what, len(cvs)))
    out = []
    for kind, atoms in cvs:
        if kind not in _CV_TYPES:
            raise ValueError("a CV is 'distance', 'angle' or 'dihedral': %r" % (kind,))
        atoms = tuple(int(a) for a in atoms)
        if len(atoms) != _CV_TYPES[kind] + 2:
            raise ValueError('a %s takes %d atoms: %s' % (kind, _CV_TYPES[kind] + 2, atoms))
        out.append((kind, atoms))
    return out


def _cv_arrays(cvs):
    """the C ABI's cv_type (n_cv,) int32 and cv_atoms (n_cv, 4) int64 of a _cv_list"""
    types = np.array([_CV_TYPES[k] for k, _ in cvs], dtype=np.int32)
    atoms = np.zeros((len(cvs), 4), dtype=np.int64)
    for j, (_, a) in enumerate(cvs):
        atoms[j, :len(a)] = a
    return types, atoms


class GDMLMetadynamics(GDMLDynamics):
    """Well-tempered multiple-walker metadynamics (Raiteri et al., J. Phys. Chem. B 110, 3533 (2006); Barducci, Bussi &
    Parrinello, PRL 100, 020603 (2008)) on the device (``sgdml_b200_metad_*``), in the units of ``GDMLDynamics``.
    `n_groups` groups of `n_walkers` Langevin walkers each: the walkers of a group deposit Gaussian hills into one
    store and are all biased by it; groups never see each other's hills, so independent groups give error bars.
    Walker w of group g is replica g n_walkers + w of the engine's handle.

    cvs: 1 to 4 collective variables, each ('distance', (i, j)), ('angle', (i, j, k)) or ('dihedral', (i, j, k, l)),
    in Angstrom or radians: |r_j - r_i|, the angle at j in [0, pi], the dihedral i-j-k-l in (-pi, pi], on plain
    coordinate differences (positions are never wrapped).  ``set_state(positions, velocities=None, step=0)``:
    positions (n_groups, n_walkers, N, 3), or (n_groups, N, 3) / (N, 3) copied to every walker (and group).
    ``run(n_steps, dt_fs, temperature_K, friction_per_fs, height_eV, widths, pace, bias_factor=inf, seed=0, stride=0)``
    integrates with BAOAB Langevin under the bias and deposits on every `pace`-th state a hill of the given widths (one
    per CV, Angstrom or radians) and height height_eV exp(-V / ((bias_factor - 1) kT)); bias_factor = inf is plain
    metadynamics, and bias_factor <= 1 is refused.  It returns ``GDMLDynamics.run``'s frames shaped (n_frames, n_groups,
    n_walkers, ...), with the model's potential energy, plus 'cv' (n_frames, n_groups, n_walkers, n_cv) and
    'bias_energy' (n_frames, n_groups, n_walkers) in eV, of the frame's state.  A hill becomes visible to the next
    state's evaluation; a run continued over several calls is one long run.  ``get_state()`` adds 'cv', 'bias_energy'
    and 'bias_forces' (eV/Angstrom); its 'forces' and 'potential_energy' are the model's.  ``hills()`` gives per group
    {'centers', 'widths' (n_hills, n_cv), 'heights' (n_hills,)} in Angstrom/radians and eV, and ``set_hills`` takes
    the same list to restart.  ``free_energy(grid)``: -bias_factor / (bias_factor - 1) V(s) (-V(s) for plain
    metadynamics) per group, shifted to a minimum of zero, in eV.  NumPy arrays or float64 CUDA tensors in, the same kind
    out."""

    def __init__(self, model, masses, cvs, n_walkers=1, n_groups=1, E_to_eV=_KCAL_PER_MOL_IN_EV,
                 F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.n_walkers = int(n_walkers)
        self.n_groups = int(n_groups)
        if self.n_walkers < 1 or self.n_groups < 1:
            raise ValueError('n_walkers and n_groups must be >= 1')
        self.cvs = _cv_list(cvs, 'metadynamics')
        self.n_cv = len(self.cvs)
        self.bias_factor = np.inf  # of the last run: free_energy's default
        super().__init__(model, masses, self.n_groups * self.n_walkers, E_to_eV, F_to_eV_Ang)
        # Angstrom or radian -> the engine's CV unit (model length or radian)
        self._cv_unit = np.array([self.Ang_to_R if k == 'distance' else 1.0 for k, _ in self.cvs])
        self._periodic = np.array([k == 'dihedral' for k, _ in self.cvs])

    def _create_handle(self):
        types, atoms = _cv_arrays(self.cvs)
        handle = ctypes.c_void_p()
        _lib.check(
            _lib.lib().sgdml_b200_metad_create(ctypes.byref(handle), self.gdml_predict._handle, self.n_groups,
                                               self.n_walkers, _lib.ptr(self.inv_mass), self.n_cv, _lib.ptr(types),
                                               _lib.ptr(atoms)),
            'metad_create',
        )
        return handle

    @property
    def _shape(self):
        return (self.n_groups, self.n_walkers)

    def _like(self, v, x):
        """the NumPy array v as x's kind (a tensor on x's device for a torch x)"""
        if hasattr(x, 'data_ptr'):
            import torch

            return torch.as_tensor(v, device=x.device)
        return v

    # ------------------------------------------------------------------ model units (L, model energy, fs)
    def _run_raw(self, n_steps, dt, gamma, kT, w0, widths, pace, dkT=np.inf, seed=0, stride=0,
                 frames=('R', 'V', 'E_pot', 'E_kin', 'cv', 'bias')):
        n_steps, stride = int(n_steps), int(stride)
        out = self._frames(n_steps, stride, frames)
        if 'cv' in out:
            out['cv'] = self._empty(tuple(out['cv'].shape) + (self.n_cv,))
        widths = np.ascontiguousarray(widths, dtype=np.float64).ravel()
        if widths.shape != (self.n_cv,):
            raise ValueError('widths must hold one value per CV: %d' % self.n_cv)
        _lib.check(
            _lib.lib().sgdml_b200_metad_run(self._handle, n_steps, float(dt), float(gamma), float(kT), float(w0),
                                            _lib.ptr(widths), int(pace), float(dkT), int(seed), stride,
                                            *(_lib.ptr(out.get(k)) for k in ('R', 'V', 'E_pot', 'E_kin', 'cv', 'bias')),
                                            _lib.current_stream()),
            'metad_run',
        )
        return out

    def _get_bias_raw(self):
        """{'cv' (n_replicas, n_cv), 'V' (n_replicas,), 'F' (n_replicas, 3N)} in model units."""
        n = self.n_replicas
        out = {'cv': self._empty((n, self.n_cv)), 'V': self._empty((n,)), 'F': self._empty((n, 3 * self.n_atoms))}
        _lib.check(_lib.lib().sgdml_b200_metad_get_bias(self._handle, _lib.ptr(out['cv']), _lib.ptr(out['V']),
                                                        _lib.ptr(out['F']), _lib.current_stream()), 'metad_get_bias')
        return out

    def _get_hills_raw(self):
        """(n_hills (n_groups,) int64, centers, widths (H, n_cv), heights (H,)), host arrays in model units."""
        n = np.zeros(self.n_groups, dtype=np.int64)
        L = _lib.lib()
        _lib.check(L.sgdml_b200_metad_get_hills(self._handle, _lib.ptr(n), None, None, None, _lib.current_stream()),
                   'metad_get_hills')
        H = int(n.sum())
        c, w, h = np.empty((H, self.n_cv)), np.empty((H, self.n_cv)), np.empty(H)
        _lib.check(L.sgdml_b200_metad_get_hills(self._handle, _lib.ptr(n), _lib.ptr(c), _lib.ptr(w), _lib.ptr(h),
                                                _lib.current_stream()), 'metad_get_hills')
        return n, c, w, h

    def _set_hills_raw(self, n_hills, centers, widths, heights):
        n = np.ascontiguousarray(n_hills, dtype=np.int64).ravel()
        H = int(n.sum()) if n.size else 0
        c = np.ascontiguousarray(centers, dtype=np.float64).reshape(H, self.n_cv)
        w = np.ascontiguousarray(widths, dtype=np.float64).reshape(H, self.n_cv)
        h = np.ascontiguousarray(heights, dtype=np.float64).reshape(H)
        if n.shape != (self.n_groups,):
            raise ValueError('n_hills must hold one count per group: %d' % self.n_groups)
        _lib.check(_lib.lib().sgdml_b200_metad_set_hills(self._handle, _lib.ptr(n), _lib.ptr(c), _lib.ptr(w),
                                                         _lib.ptr(h), _lib.current_stream()), 'metad_set_hills')

    # ------------------------------------------------------------------ ASE units
    def set_state(self, positions, velocities=None, step=0):
        axes = ('n_groups', 'n_walkers')
        positions = _groups(positions, 'positions', self.n_groups, self.n_walkers, self.n_atoms, axes)
        if velocities is not None:
            velocities = _groups(velocities, 'velocities', self.n_groups, self.n_walkers, self.n_atoms, axes)
        super().set_state(positions, velocities, step)

    def get_state(self):
        out = super().get_state()
        b = self._get_bias_raw()
        g = self._shape
        out.update(cv=(b['cv'] / self._like(self._cv_unit, b['cv'])).reshape(g + (self.n_cv,)),
                   bias_energy=(b['V'] * self.E_to_eV).reshape(g),
                   bias_forces=(b['F'] * self.F_to_eV_Ang).reshape(g + (self.n_atoms, 3)))
        return out

    def run(self, n_steps, dt_fs, temperature_K, friction_per_fs, height_eV, widths, pace, bias_factor=np.inf, seed=0,
            stride=0):
        bias_factor = float(bias_factor)
        if not bias_factor > 1.0:
            raise ValueError('bias_factor must be > 1 (inf: plain metadynamics): %r' % bias_factor)
        kT = KB_EV * float(temperature_K) / self.E_to_eV
        dkT = np.inf if np.isinf(bias_factor) else (bias_factor - 1.0) * kT
        w = np.asarray(widths, dtype=np.float64).ravel() * self._cv_unit
        f = self._run_raw(n_steps, dt_fs, friction_per_fs, kT, float(height_eV) / self.E_to_eV, w, pace, dkT, seed,
                          stride)
        self.bias_factor = bias_factor
        out = self._ase_frames(f)
        if 'cv' in f:
            nf = f['cv'].shape[0]
            out['cv'] = (f['cv'] / self._like(self._cv_unit, f['cv'])).reshape((nf,) + self._shape + (self.n_cv,))
            out['bias_energy'] = (f['bias'] * self.E_to_eV).reshape((nf,) + self._shape)
        return out

    def hills(self):
        """[{'centers', 'widths': (n_hills, n_cv), 'heights': (n_hills,)}] per group, Angstrom/radians and eV (NumPy)."""
        n, c, w, h = self._get_hills_raw()
        edges = np.concatenate([[0], np.cumsum(n)])
        return [{'centers': c[a:b] / self._cv_unit, 'widths': w[a:b] / self._cv_unit, 'heights': h[a:b] * self.E_to_eV}
                for a, b in zip(edges[:-1], edges[1:])]

    def set_hills(self, hills):
        """Replaces every group's hills with `hills`, a list of one dict per group as ``hills()`` gives them."""
        if len(hills) != self.n_groups:
            raise ValueError('hills must hold one entry per group: %d' % self.n_groups)
        parts = [(np.asarray(g['centers'], dtype=np.float64).reshape(-1, self.n_cv) * self._cv_unit,
                  np.asarray(g['widths'], dtype=np.float64).reshape(-1, self.n_cv) * self._cv_unit,
                  np.asarray(g['heights'], dtype=np.float64).ravel() / self.E_to_eV) for g in hills]
        n = [len(p[2]) for p in parts]
        cat = [np.concatenate([p[i] for p in parts]) if sum(n) else np.empty((0,) + parts[0][i].shape[1:])
               for i in range(3)]
        self._set_hills_raw(n, *cat)

    def bias(self, grid):
        """V(s) (eV) per group on the grid: (n_groups, n) for one CV and a grid of n points, (n_groups, n0, n1) for two
        CVs and a grid (g0, g1) of n0 and n1 points (Angstrom or radians), summed from ``hills()`` in NumPy."""
        if self.n_cv == 1:
            pts = np.asarray(grid, dtype=np.float64).reshape(-1, 1)
            shape = (pts.shape[0],)
        elif self.n_cv == 2:
            g0, g1 = (np.asarray(g, dtype=np.float64).ravel() for g in grid)
            pts = np.stack(np.meshgrid(g0, g1, indexing='ij'), -1).reshape(-1, 2)
            shape = (len(g0), len(g1))
        else:
            raise ValueError('free_energy and bias take a grid over 1 or 2 CVs, not %d' % self.n_cv)
        out = []
        for g in self.hills():
            d = pts[:, None, :] - g['centers'][None]
            d = np.where(self._periodic, (d + np.pi) % (2.0 * np.pi) - np.pi, d)
            a = ((d / g['widths'][None]) ** 2).sum(-1)
            out.append((g['heights'][None] * np.exp(-0.5 * a)).sum(-1).reshape(shape))
        return np.array(out)

    def free_energy(self, grid, bias_factor=None):
        """-bias_factor / (bias_factor - 1) V(s) per group (eV; -V(s) for bias_factor = inf), shifted so that each
        group's minimum is zero; grid and shape as ``bias``.  bias_factor: that of the last run by default."""
        gamma = self.bias_factor if bias_factor is None else float(bias_factor)
        f = -self.bias(grid) * (1.0 if np.isinf(gamma) else gamma / (gamma - 1.0))
        return f - f.reshape(self.n_groups, -1).min(1).reshape((self.n_groups,) + (1,) * (f.ndim - 1))


class GDMLUmbrellaSampling(GDMLDynamics):
    """Umbrella sampling with Hamiltonian replica exchange between neighbouring windows (REUS; Sugita, Kitao & Okamoto,
    J. Chem. Phys. 113, 6042 (2000)) on the device (``sgdml_b200_umbrella_*``), reweighted by MBAR (Shirts & Chodera,
    J. Chem. Phys. 129, 124105 (2008)), in the units of ``GDMLDynamics``.  `n_ladders` independent ladders of
    n_windows Langevin replicas: slot k of ladder l (replica l n_windows + k of the engine's handle) is restrained by
    window k for the whole run, and neighbouring windows swap configurations by the Metropolis test on the restraint
    energies, inside the step graph.  Independent ladders give error bars.

    cvs: 1 to 4 CVs as ``GDMLMetadynamics`` takes them (Angstrom or radians).  centers, force_constants:
    (n_windows, n_cv) (or (n_windows,) for one CV): window k adds sum_j 0.5 kappa_kj (s_j - c_kj)^2, kappa in eV/Angstrom^2
    or eV/rad^2, a dihedral's difference wrapped into [-pi, pi) and its centre in (-pi, pi].
    ``set_state(positions, velocities=None, step=0)``: positions (n_ladders, n_windows, N, 3), or (n_ladders, N, 3) /
    (N, 3) copied to every window (and ladder); it resets the walker labels to the slots.  ``get_state()`` adds 'cv',
    'bias_energy' and 'bias_forces'; its 'forces' and 'potential_energy' are the model's.  ``set_windows(centers,
    force_constants)`` replaces the windows.
    ``run(n_steps, dt_fs, temperature_K, friction_per_fs, exchange_every=0, seed=0, stride=0)`` returns
    ``GDMLReplicaExchange.run``'s keys shaped (..., n_ladders, n_windows, ...), plus 'cv' (n_frames, n_ladders,
    n_windows, n_cv) and 'bias_energy' (eV) of every frame's state after its exchange.  A run continued over several
    calls is one long run.
    ``mbar(cv_frames, temperature_K, windows=None, tol=1e-10, max_iter=10000)`` reweights `cv_frames` (run's 'cv', slot k
    of every frame a sample of window k) per ladder on the device: [{'f' (n_windows,) the window free energies in eV
    with f[0] = 0, 'log_w' (n_frames, n_windows) the log unbiased weight of each sample (they sum to 1), 'n_iter',
    'resid' (the last max |df| in units of kT)}].  windows: (centers, force_constants) of the frames, default the
    handle's.  ``free_energy(cv_frames, bins, temperature_K, windows=None)``: the profile -kT ln sum_{n in bin} w_n
    (eV) per ladder, shifted to a minimum of zero, NaN for empty bins: bins are the edges along CV 0, or a pair of edge
    arrays along CVs 0 and 1; the other CVs are marginalised.  NumPy arrays or float64 CUDA tensors in, the same kind
    out."""

    def __init__(self, model, masses, cvs, centers, force_constants, n_ladders=1, E_to_eV=_KCAL_PER_MOL_IN_EV,
                 F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.cvs = _cv_list(cvs, 'umbrella sampling')
        self.n_cv = len(self.cvs)
        self._windows_arg = (centers, force_constants)
        self.n_windows = len(self._window_arrays(centers, force_constants)[0])
        self.n_ladders = int(n_ladders)
        if self.n_ladders < 1 or self.n_windows < 1:
            raise ValueError('n_ladders and the number of windows must be >= 1')
        self._periodic = np.array([k == 'dihedral' for k, _ in self.cvs])
        super().__init__(model, masses, self.n_ladders * self.n_windows, E_to_eV, F_to_eV_Ang)

    @property
    def _cv_unit(self):
        """Angstrom or radian -> the engine's CV unit (model length or radian)"""
        return np.array([self.Ang_to_R if k == 'distance' else 1.0 for k, _ in self.cvs])

    def _window_arrays(self, centers, force_constants):
        """(centers, force constants) as (n_windows, n_cv) float64 arrays in the caller's units"""
        c = np.asarray(_host(centers), dtype=np.float64)
        k = np.asarray(_host(force_constants), dtype=np.float64)
        c = c.reshape(-1, 1) if c.ndim == 1 and self.n_cv == 1 else c
        k = k.reshape(-1, 1) if k.ndim == 1 and self.n_cv == 1 else k
        if c.ndim != 2 or c.shape[1] != self.n_cv or k.shape != c.shape:
            raise ValueError('centers and force_constants must be (n_windows, n_cv) with n_cv = %d: %s, %s'
                             % (self.n_cv, c.shape, k.shape))
        return c, k

    def _raw_windows(self, centers, force_constants):
        """the window table in model units: centres in L or rad, force constants in model energy / L^2 or / rad^2"""
        c, k = self._window_arrays(centers, force_constants)
        if c.shape[0] != getattr(self, 'n_windows', c.shape[0]):
            raise ValueError('the windows must number %d: %d' % (self.n_windows, c.shape[0]))
        u = self._cv_unit
        return np.ascontiguousarray(c * u), np.ascontiguousarray(k / self.E_to_eV / (u * u))

    def _create_handle(self):
        types, atoms = _cv_arrays(self.cvs)
        c, k = self._raw_windows(*self._windows_arg)
        self.windows = self._window_arrays(*self._windows_arg)
        handle = ctypes.c_void_p()
        _lib.check(
            _lib.lib().sgdml_b200_umbrella_create(ctypes.byref(handle), self.gdml_predict._handle, self.n_ladders,
                                                  self.n_windows, _lib.ptr(self.inv_mass), self.n_cv, _lib.ptr(types),
                                                  _lib.ptr(atoms), _lib.ptr(c), _lib.ptr(k)),
            'umbrella_create',
        )
        return handle

    @property
    def _shape(self):
        return (self.n_ladders, self.n_windows)

    def _like(self, v, x):
        return GDMLMetadynamics._like(self, v, x)

    # ------------------------------------------------------------------ model units (L, model energy, fs)
    def _set_windows_raw(self, centers, kappas):
        c = np.ascontiguousarray(centers, dtype=np.float64)
        k = np.ascontiguousarray(kappas, dtype=np.float64)
        if c.size != self.n_windows * self.n_cv or k.size != c.size:
            raise ValueError('centers and kappas must hold n_windows x n_cv = %d x %d values each'
                             % (self.n_windows, self.n_cv))
        _lib.check(_lib.lib().sgdml_b200_umbrella_set_windows(self._handle, _lib.ptr(c), _lib.ptr(k),
                                                              _lib.current_stream()), 'umbrella_set_windows')

    def _run_raw(self, n_steps, dt, gamma, kT, exchange_every=0, seed=0, stride=0,
                 frames=('R', 'V', 'E_pot', 'E_kin', 'cv', 'bias', 'walker')):
        """-> frames, 'walkers' (n_replicas,), 'n_accepted', 'n_attempted' (n_ladders, n_windows - 1)."""
        n_steps, stride = int(n_steps), int(stride)
        out = self._frames(n_steps, stride, frames)
        if 'cv' in out:
            out['cv'] = self._empty(tuple(out['cv'].shape) + (self.n_cv,))
        walkers = self._empty((self.n_replicas,), np.int32)
        acc, att = (self._empty((self.n_ladders, self.n_windows - 1), np.int64) for _ in range(2))
        _lib.check(
            _lib.lib().sgdml_b200_umbrella_run(self._handle, n_steps, float(dt), float(gamma), float(kT), int(seed),
                                               int(exchange_every), stride,
                                               *(_lib.ptr(out.get(k)) for k in ('R', 'V', 'E_pot', 'E_kin', 'cv', 'bias',
                                                                               'walker')),
                                               _lib.ptr(walkers), _lib.ptr(acc), _lib.ptr(att), _lib.current_stream()),
            'umbrella_run',
        )
        out.update(walkers=walkers, n_accepted=acc, n_attempted=att)
        return out

    def _get_bias_raw(self):
        """{'cv' (n_replicas, n_cv), 'V' (n_replicas,), 'F' (n_replicas, 3N)} in model units."""
        n = self.n_replicas
        out = {'cv': self._empty((n, self.n_cv)), 'V': self._empty((n,)), 'F': self._empty((n, 3 * self.n_atoms))}
        _lib.check(_lib.lib().sgdml_b200_umbrella_get_bias(self._handle, _lib.ptr(out['cv']), _lib.ptr(out['V']),
                                                           _lib.ptr(out['F']), _lib.current_stream()),
                   'umbrella_get_bias')
        return out

    def _mbar_raw(self, samples, n_per_window, beta, centers, kappas, tol=1e-10, max_iter=10000):
        """MBAR over samples (n, n_cv) in model units (NumPy or a float64 CUDA tensor), pooled window after window.
        -> (f (K,), log_w (n,) of the samples' kind, n_iter, resid)."""
        n = int(samples.shape[0])
        counts = np.ascontiguousarray(n_per_window, dtype=np.int64)
        c = np.ascontiguousarray(centers, dtype=np.float64)
        k = np.ascontiguousarray(kappas, dtype=np.float64)
        types, _ = _cv_arrays(self.cvs)
        if hasattr(samples, 'data_ptr'):
            _check_cuda_f64(samples, 'samples')
            import torch

            samples = samples.contiguous()
            f = torch.empty(len(counts), dtype=torch.float64, device=samples.device)
            log_w = torch.empty(n, dtype=torch.float64, device=samples.device)
        else:
            samples = np.ascontiguousarray(samples, dtype=np.float64)
            f, log_w = np.empty(len(counts)), np.empty(n)
        n_iter, resid = np.zeros(1, dtype=np.int64), np.zeros(1)
        _lib.check(
            _lib.lib().sgdml_b200_umbrella_mbar(len(counts), self.n_cv, _lib.ptr(types), _lib.ptr(c), _lib.ptr(k),
                                                float(beta), n, _lib.ptr(samples), _lib.ptr(counts), float(tol),
                                                int(max_iter), _lib.ptr(f), _lib.ptr(log_w), _lib.ptr(n_iter),
                                                _lib.ptr(resid), _lib.current_stream()),
            'umbrella_mbar',
        )
        return f, log_w, int(n_iter[0]), float(resid[0])

    # ------------------------------------------------------------------ ASE units
    def set_state(self, positions, velocities=None, step=0):
        axes = ('n_ladders', 'n_windows')
        positions = _groups(positions, 'positions', self.n_ladders, self.n_windows, self.n_atoms, axes)
        if velocities is not None:
            velocities = _groups(velocities, 'velocities', self.n_ladders, self.n_windows, self.n_atoms, axes)
        super().set_state(positions, velocities, step)

    def get_state(self):
        out = super().get_state()
        b = self._get_bias_raw()
        g = self._shape
        out.update(cv=(b['cv'] / self._like(self._cv_unit, b['cv'])).reshape(g + (self.n_cv,)),
                   bias_energy=(b['V'] * self.E_to_eV).reshape(g),
                   bias_forces=(b['F'] * self.F_to_eV_Ang).reshape(g + (self.n_atoms, 3)))
        return out

    def set_windows(self, centers, force_constants):
        self._set_windows_raw(*self._raw_windows(centers, force_constants))
        self.windows = self._window_arrays(centers, force_constants)

    def run(self, n_steps, dt_fs, temperature_K, friction_per_fs, exchange_every=0, seed=0, stride=0):
        kT = KB_EV * float(temperature_K) / self.E_to_eV
        f = self._run_raw(n_steps, dt_fs, friction_per_fs, kT, exchange_every, seed, stride)
        acc, att = f['n_accepted'], f['n_attempted']
        ratio = acc.double() / att.clip(1).double() if hasattr(att, 'data_ptr') else acc / att.clip(1)
        ratio[att == 0] = np.nan
        out = {'walkers': f['walkers'].reshape(self._shape), 'n_accepted': acc, 'n_attempted': att, 'acceptance': ratio}
        out.update(self._ase_frames(f))
        if 'walker' in f:
            nf = f['walker'].shape[0]
            out['walker'] = f['walker'].reshape((nf,) + self._shape)
            out['cv'] = (f['cv'] / self._like(self._cv_unit, f['cv'])).reshape((nf,) + self._shape + (self.n_cv,))
            out['bias_energy'] = (f['bias'] * self.E_to_eV).reshape((nf,) + self._shape)
        return out

    def mbar(self, cv_frames, temperature_K, windows=None, tol=1e-10, max_iter=10000):
        kT_eV = KB_EV * float(temperature_K)
        c, k = self._raw_windows(*(windows if windows is not None else self.windows))
        x = cv_frames
        if tuple(x.shape[1:]) != self._shape + (self.n_cv,):
            raise ValueError('cv_frames must be (n_frames, n_ladders, n_windows, n_cv) = (n, %d, %d, %d): %s'
                             % (self._shape + (self.n_cv, tuple(x.shape))))
        nf = int(x.shape[0])
        x = x * self._like(self._cv_unit, x)
        out = []
        for l in range(self.n_ladders):
            s = x[:, l].transpose(1, 0, 2) if not hasattr(x, 'data_ptr') else x[:, l].permute(1, 0, 2)
            s = s.reshape(self.n_windows * nf, self.n_cv)
            f, log_w, n_iter, resid = self._mbar_raw(s, [nf] * self.n_windows, self.E_to_eV / kT_eV, c, k, tol,
                                                      max_iter)
            out.append({'f': f * kT_eV, 'log_w': log_w.reshape(self.n_windows, nf).T, 'n_iter': n_iter,
                        'resid': resid})
        return out

    def free_energy(self, cv_frames, bins, temperature_K, windows=None):
        kT_eV = KB_EV * float(temperature_K)
        edges = [np.asarray(_host(b), dtype=np.float64).ravel() for b in
                 (bins if isinstance(bins, (tuple, list)) and np.ndim(bins[0]) == 1 else [bins])]
        if not 1 <= len(edges) <= min(2, self.n_cv):
            raise ValueError('free_energy takes bin edges along 1 or 2 CVs (at most n_cv = %d)' % self.n_cv)
        x = np.asarray(_host(cv_frames), dtype=np.float64)
        out = []
        for r in self.mbar(cv_frames, temperature_K, windows):
            w = np.exp(np.asarray(_host(r['log_w'])))  # (n_frames, n_windows)
            h, _ = np.histogramdd(x[:, len(out)].reshape(-1, self.n_cv)[:, :len(edges)], bins=edges,
                                  weights=w.reshape(-1))
            with np.errstate(divide='ignore'):
                F = np.where(h > 0, -kT_eV * np.log(np.where(h > 0, h, 1.0)), np.nan)
            out.append(F - np.nanmin(F))
        return self._like(np.array(out), cv_frames)


def _host(x):
    """a NumPy view of x (a CUDA tensor is copied to the host)"""
    return x.detach().cpu().numpy() if hasattr(x, 'data_ptr') else x


def _det3(a):
    """det of (..., 3, 3) NumPy arrays or torch tensors, by cofactors of the first row."""
    return (a[..., 0, 0] * (a[..., 1, 1] * a[..., 2, 2] - a[..., 1, 2] * a[..., 2, 1])
            - a[..., 0, 1] * (a[..., 1, 0] * a[..., 2, 2] - a[..., 1, 2] * a[..., 2, 0])
            + a[..., 0, 2] * (a[..., 1, 0] * a[..., 2, 1] - a[..., 1, 1] * a[..., 2, 0]))


class GDMLRelaxation(GDMLDynamics):
    """Relaxes `n_replicas` geometries of one model to local minima of its energy, on the device, with FIRE or L-BFGS.

    The handle is an MD handle with unit inverse masses, which the optimisers never read; ``set_state`` and
    ``get_state`` are ``GDMLDynamics``'s, and ``run`` raises (there are no masses to integrate with).  ``relax(positions=None, fmax=0.05, max_steps=1000, optimizer='lbfgs',
    maxstep=0.2, memory=20, alpha=70.0, dt=0.1, dtmax=1.0)`` relaxes from `positions` ((n_replicas, N, 3) or (N, 3) for
    one replica, Angstrom; None: the current state) until every replica has max_a |F_a| < fmax (eV/Angstrom, ASE's
    criterion) or max_steps steps have run, and returns {'positions', 'forces' (n_replicas, N, 3), 'potential_energy',
    'fmax' (n_replicas,), 'converged' (n_replicas,) bool, 'n_steps' (n_replicas,) int64} in Angstrom, eV/Angstrom and
    eV.  The arguments and defaults are those of ASE's optimisers: maxstep in Angstrom (FIRE: the whole step, L-BFGS:
    each atom's); L-BFGS keeps `memory` pairs (1 to 32) and starts from the inverse Hessian 1/alpha (Angstrom^2/eV);
    FIRE starts at time step dt and grows it up to dtmax (ASE's time unit).  Every call starts afresh, as a new ASE
    optimiser would; afterwards the velocities are zero and the step index is unchanged.  NumPy arrays or float64 CUDA
    tensors in, the same kind out."""

    def __init__(self, model, n_replicas=1, E_to_eV=_KCAL_PER_MOL_IN_EV, F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self._init_model(model, n_replicas, E_to_eV, F_to_eV_Ang)
        self.inv_mass = np.ones(self.n_atoms)
        self._handle = self._create_handle()

    def run(self, *args, **kwargs):
        """Not available: the handle's inverse masses are ones in model units, not the masses ``GDMLDynamics.run``
        integrates with.  Run MD on relaxed geometries with a ``GDMLDynamics`` of the real masses."""
        raise TypeError('GDMLRelaxation has no MD run: pass the relaxed positions to GDMLDynamics(model, masses)')

    # ------------------------------------------------------------------ model units
    def _relax_raw(self, optimizer, max_steps, fmax, maxstep, *args):
        """FIRE: args = (dt, dtmax); L-BFGS: args = (memory, h0), all in model units.  -> (n_steps, converged, fmax)."""
        n = self.n_replicas
        out = (self._empty(n, np.int64), self._empty(n, np.int32), self._empty(n))
        L = _lib.lib()
        if optimizer == 'fire':
            rc = L.sgdml_b200_relax_fire(self._handle, int(max_steps), float(fmax), float(maxstep), float(args[0]),
                                         float(args[1]), *(_lib.ptr(x) for x in out), _lib.current_stream())
        elif optimizer == 'lbfgs':
            rc = L.sgdml_b200_relax_lbfgs(self._handle, int(max_steps), float(fmax), float(maxstep), int(args[0]),
                                          float(args[1]), *(_lib.ptr(x) for x in out), _lib.current_stream())
        else:
            raise ValueError("optimizer must be 'lbfgs' or 'fire': %r" % (optimizer,))
        _lib.check(rc, 'relax_' + optimizer)
        return out

    # ------------------------------------------------------------------ ASE units
    def relax(self, positions=None, fmax=0.05, max_steps=1000, optimizer='lbfgs', maxstep=0.2, memory=20, alpha=70.0,
              dt=0.1, dtmax=1.0):
        if optimizer not in ('lbfgs', 'fire'):
            raise ValueError("optimizer must be 'lbfgs' or 'fire': %r" % (optimizer,))
        if positions is not None:
            self.set_state(positions)
        c = self.Ang_to_R * self.F_to_eV_Ang  # dt^2 and the inverse Hessian: Angstrom^2 / eV -> model units
        if optimizer == 'fire':
            args = (float(dt) * np.sqrt(c), float(dtmax) * np.sqrt(c))
        else:
            args = (memory, c / float(alpha))
        n_steps, conv, fm = self._relax_raw(optimizer, max_steps, float(fmax) / self.F_to_eV_Ang,
                                            float(maxstep) * self.Ang_to_R, *args)
        st = self.get_state()
        return {'positions': st['positions'], 'forces': st['forces'], 'potential_energy': st['potential_energy'],
                'fmax': fm * self.F_to_eV_Ang, 'converged': conv != 0, 'n_steps': n_steps}


class GDMLNEB(GDMLRelaxation):
    """Minimum-energy paths and saddle points of one model with the nudged elastic band (NEB) and its climbing-image
    form (CI-NEB), optimised on the device (``sgdml_b200_neb_fire``): `n_bands` bands of `n_images` images (>= 3),
    many bands and many steps per call.  Image j of band b is replica b n_images + j of a ``GDMLRelaxation`` handle;
    images 0 and n_images - 1 are the fixed endpoints.  Image differences are plain coordinate differences, with no
    minimum image, also for periodic models.

    ``neb(images=None, fmax=0.05, max_steps=1000, k=0.1, climb=False, maxstep=0.2, dt=0.1, dtmax=1.0)`` runs FIRE on
    every band (its interior images as one vector, as ASE's optimisers on an ``NEB`` object) until max over the atoms of
    all interior images of |F_neb| < fmax, or max_steps steps.  Units are ASE's: images (n_bands, n_images, N, 3) [or
    (n_images, N, 3) for one band] in Angstrom (None: continue from the current state, so that the usual two-stage run
    is a call without `climb` and a second call with it); fmax in eV/Angstrom; the spring constant k in eV/Angstrom^2;
    maxstep (Angstrom) caps the step of a whole band; dt and dtmax as in ``GDMLRelaxation.relax``.  Returns
    {'positions', 'forces' (the model's forces): (n_bands, n_images, N, 3), 'energies': (n_bands, n_images), 'barrier':
    the highest interior energy minus that of image 0, 'climbing_image' (the highest interior image), 'fmax' (of the NEB
    forces), 'converged', 'n_steps': (n_bands,)} in Angstrom, eV/Angstrom and eV.  NumPy arrays or float64 CUDA tensors
    in, the same kind out.  ``interpolate`` builds a linear band between two endpoints."""

    def __init__(self, model, n_images, n_bands=1, E_to_eV=_KCAL_PER_MOL_IN_EV, F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.n_images = int(n_images)
        self.n_bands = int(n_bands)
        if self.n_images < 3 or self.n_bands < 1:
            raise ValueError('a band needs n_images >= 3 (two endpoints and an interior image), and n_bands >= 1')
        super().__init__(model, self.n_bands * self.n_images, E_to_eV, F_to_eV_Ang)

    def interpolate(self, initial, final, n_images=None, align=True):
        """Linear band from `initial` to `final` (host arrays (..., N, 3), Angstrom): (..., n_images, N, 3), image 0
        exactly `initial` and the last image exactly the (aligned) `final`.  align: first move `final` onto `initial`
        by the rigid rotation and translation of least squares (Kabsch), which a periodic model refuses."""
        if align and self.gdml_predict.lat_and_inv is not None:
            raise ValueError('align=True moves the atoms rigidly, which a periodic model does not allow: pass align=False')
        n_images = self.n_images if n_images is None else int(n_images)
        if n_images < 2:
            raise ValueError('n_images must be >= 2')
        a = np.asarray(initial, dtype=np.float64)
        b = np.asarray(final, dtype=np.float64)
        if a.shape != b.shape or a.ndim < 2 or a.shape[-1] != 3:
            raise ValueError('initial and final must have the same shape (..., N, 3): %s, %s' % (a.shape, b.shape))
        if align:
            b = kabsch_align(b, a)
        t = (np.arange(n_images, dtype=np.float64) / (n_images - 1)).reshape(n_images, 1, 1)
        out = a[..., None, :, :] + t * (b - a)[..., None, :, :]
        out[..., 0, :, :] = a
        out[..., -1, :, :] = b
        return out

    def _bands(self, x):
        """(n_bands, n_images, N, 3) or (n_images, N, 3) for one band."""
        shape = tuple(x.shape)
        want = (self.n_bands, self.n_images, self.n_atoms, 3)
        if shape != want and not (self.n_bands == 1 and shape == want[1:]):
            raise ValueError('images must be (n_bands, n_images, N, 3) = %s, or (n_images, N, 3) for one band: %s'
                             % (want, shape))
        return x

    # ------------------------------------------------------------------ model units
    def _neb_raw(self, max_steps, fmax, k, climb, maxstep, dt, dtmax):
        """-> (n_steps, converged, fmax, climbing_image), each (n_bands,), in model units."""
        n = self.n_bands
        out = (self._empty(n, np.int64), self._empty(n, np.int32), self._empty(n), self._empty(n, np.int32))
        _lib.check(
            _lib.lib().sgdml_b200_neb_fire(self._handle, self.n_images, int(max_steps), float(fmax), float(k),
                                           1 if climb else 0, float(maxstep), float(dt), float(dtmax),
                                           *(_lib.ptr(x) for x in out), _lib.current_stream()),
            'neb_fire',
        )
        return out

    # ------------------------------------------------------------------ ASE units
    def neb(self, images=None, fmax=0.05, max_steps=1000, k=0.1, climb=False, maxstep=0.2, dt=0.1, dtmax=1.0):
        if images is not None:
            self.set_state(self._bands(images))
        c = self.Ang_to_R * self.F_to_eV_Ang  # eV / Angstrom^2 -> model force / model length, and dt^2
        n_steps, conv, fm, top = self._neb_raw(max_steps, float(fmax) / self.F_to_eV_Ang, float(k) / c, climb,
                                               float(maxstep) * self.Ang_to_R, float(dt) * np.sqrt(c),
                                               float(dtmax) * np.sqrt(c))
        st = self.get_state()
        shape = (self.n_bands, self.n_images)
        E = st['potential_energy'].reshape(shape)
        inner = E[:, 1:-1]
        top_E = inner.amax(1) if hasattr(inner, 'data_ptr') else inner.max(1)
        return {'positions': st['positions'].reshape(shape + (self.n_atoms, 3)),
                'forces': st['forces'].reshape(shape + (self.n_atoms, 3)), 'energies': E, 'barrier': top_E - E[:, 0],
                'climbing_image': top, 'fmax': fm * self.F_to_eV_Ang, 'converged': conv != 0, 'n_steps': n_steps}


class GDMLDimer(GDMLRelaxation):
    """First-order saddle points next to a minimum, with no final state, by the dimer method (Henkelman & Jonsson,
    J. Chem. Phys. 111, 7010 (1999)) on the device (``sgdml_b200_dimer_fire``): `n_dimers` independent searches, many
    steps per call.  Dimer d is replicas 2d (its centre) and 2d + 1 (its image, the centre plus `separation` along the
    dimer's unit mode) of a ``GDMLRelaxation`` handle; the mode follows the lowest-curvature direction (one rotation per
    translation at most, by the curvature fit of Heyden, Bell & Keil, J. Chem. Phys. 123, 224101 (2005)) and the centre
    moves by FIRE up that mode and down every other.  The mode is kept orthogonal to rigid translations and, for free
    molecules, rotations.

    ``search(positions=None, modes=None, fmax=0.05, max_steps=1000, separation=1e-4, trial_angle=pi/4, rot_min=0.1,
    maxstep=0.1, dt=0.1, dtmax=1.0, seed=0)`` runs until every dimer has max_a |F_a| < fmax at its centre with a
    negative curvature along its mode, or `max_steps` force evaluations of the pairs (a rotating step takes two).
    Units are ASE's: positions (n_dimers, N, 3), or (N, 3) for every dimer, in Angstrom (None: continue from the
    current centres); modes (n_dimers, N, 3) or (N, 3), any length (None: keep the modes of the previous call, or on
    the first call Gaussian modes from ``numpy.random.default_rng(seed)``); fmax in eV/Angstrom; separation and maxstep
    (the centre's whole step) in Angstrom; rot_min, the rotational force below which a dimer translates without
    rotating, in eV/Angstrom^2; dt and dtmax as in ``GDMLRelaxation.relax``.  Returns, for the centres, {'positions',
    'forces', 'mode' (unit, (n_dimers, N, 3)), 'potential_energy', 'curvature' (eV/Angstrom^2, along the final mode),
    'fmax', 'converged', 'n_steps' (translations), 'n_rotations': (n_dimers,)}.  NumPy arrays or float64 CUDA tensors
    in, the same kind out."""

    def __init__(self, model, n_dimers=1, E_to_eV=_KCAL_PER_MOL_IN_EV, F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.n_dimers = int(n_dimers)
        if self.n_dimers < 1:
            raise ValueError('n_dimers must be >= 1')
        self._has_modes = False
        super().__init__(model, 2 * self.n_dimers, E_to_eV, F_to_eV_Ang)

    def _per_dimer(self, x, name):
        """(n_dimers, N, 3) or (N, 3) -> (n_dimers, 3N), the same kind; torch inputs must be float64 CUDA tensors."""
        return _per_unit(x, name, self.n_dimers, self.n_atoms, 'n_dimers')

    # ------------------------------------------------------------------ model units
    def _dimer_raw(self, modes, max_steps, fmax, separation, cos_trial, sin_trial, rot_min, maxstep, dt, dtmax):
        """modes (n_dimers, 3N) or None (keep) -> (n_steps, converged, fmax, curvature, n_rot (n_dimers,), modes
        (n_dimers, 3N)), in model units."""
        n = self.n_dimers
        if modes is not None:  # the entry point copies n_dimers 3N doubles from this pointer
            if hasattr(modes, 'data_ptr'):
                _check_cuda_f64(modes, 'modes')
                modes = modes.contiguous()
            else:
                modes = np.ascontiguousarray(modes, dtype=np.float64)
            if tuple(modes.shape) != (n, 3 * self.n_atoms):
                raise ValueError('modes must be (n_dimers, 3N) = (%d, %d): %s' % (n, 3 * self.n_atoms,
                                                                                  tuple(modes.shape)))
        out = (self._empty(n, np.int64), self._empty(n, np.int32), self._empty(n), self._empty(n),
               self._empty(n, np.int64), self._empty((n, 3 * self.n_atoms)))
        _lib.check(
            _lib.lib().sgdml_b200_dimer_fire(self._handle, _lib.ptr(modes), int(max_steps), float(fmax),
                                             float(separation), float(cos_trial), float(sin_trial), float(rot_min),
                                             float(maxstep), float(dt), float(dtmax), *(_lib.ptr(x) for x in out),
                                             _lib.current_stream()),
            'dimer_fire',
        )
        self._has_modes = True
        return out

    # ------------------------------------------------------------------ ASE units
    def search(self, positions=None, modes=None, fmax=0.05, max_steps=1000, separation=1e-4, trial_angle=np.pi / 4,
               rot_min=0.1, maxstep=0.1, dt=0.1, dtmax=1.0, seed=0):
        # both are checked before the state changes
        R = None if positions is None else self._per_dimer(positions, 'positions')
        if modes is not None:
            modes = self._per_dimer(modes, 'modes')
        if R is not None:
            R = R.repeat_interleave(2, 0) if hasattr(R, 'data_ptr') else np.repeat(R, 2, axis=0)
            self.set_state(R.reshape(self.n_replicas, self.n_atoms, 3))
        if modes is None and not self._has_modes:
            modes = np.random.default_rng(seed).standard_normal((self.n_dimers, 3 * self.n_atoms))
        c = self.Ang_to_R * self.F_to_eV_Ang  # eV / Angstrom^2 -> model force / model length, and dt^2
        phi = float(trial_angle)
        n_steps, conv, fm, curv, n_rot, mode = self._dimer_raw(
            modes, max_steps, float(fmax) / self.F_to_eV_Ang, float(separation) * self.Ang_to_R, math.cos(phi),
            math.sin(phi), float(rot_min) / c, float(maxstep) * self.Ang_to_R, float(dt) * np.sqrt(c),
            float(dtmax) * np.sqrt(c))
        st = self.get_state()
        g = (self.n_dimers, self.n_atoms, 3)
        return {'positions': st['positions'][0::2].reshape(g), 'forces': st['forces'][0::2].reshape(g),
                'potential_energy': st['potential_energy'][0::2], 'mode': mode.reshape(g), 'curvature': curv * c,
                'fmax': fm * self.F_to_eV_Ang, 'converged': conv != 0, 'n_steps': n_steps, 'n_rotations': n_rot}


class GDMLIRC(GDMLRelaxation):
    """Which two minima a first-order saddle connects: the intrinsic reaction coordinate (IRC), the steepest-descent
    path in mass-weighted coordinates, followed downhill from each saddle in both directions along its imaginary mode
    on the device (``sgdml_b200_irc_rk4``), by classical RK4 with a fixed step (Schmidt, Gordon & Dupuis, JACS 107,
    2585 (1985)); `n_saddles` saddles, two branches each, many points per call.  Branch j of saddle k is replica 2k + j
    of a ``GDMLRelaxation`` handle that carries the real inverse masses (masses (N,) in amu), so the inherited ``relax``
    works on the branch ends.

    ``run(saddles, modes, step=0.05, max_points=500, fmax=0.05, relax_ends=True, relax_steps=1000)``: saddles
    (n_saddles, N, 3) or (N, 3) in Angstrom; modes of the same shape, the Cartesian displacement of each saddle's
    imaginary mode in any length (``GDMLVibrations.analyse(saddle)['modes'][:, 0]``, or a dimer's mode); step in
    amu^1/2 Angstrom (the default is close to the common 0.1 amu^1/2 bohr); fmax in eV/Angstrom.  Branch 0 follows
    +mode, branch 1 -mode.  A branch ends when a new point's energy is not below the last one's (end 2, at the last
    point), when max_a |F_a| < fmax (end 1) or at max_points points (end 3).  Returns {'positions' (n_saddles, 2,
    max_points, N, 3), 'energies' (n_saddles, 2, max_points), 's' (n_saddles, 2, max_points): the signed mass-weighted
    arc length in amu^1/2 Angstrom (+ forward, - backward), n step at point n, which RK4 integrates as the arc length;
    all NaN past the branch's point count; 'n_points', 'end', 'fmax' (n_saddles, 2)} in Angstrom and eV.  With relax_ends, L-BFGS (``relax`` at the same fmax, relax_steps steps) then
    takes the branch ends to their minima: 'minima' {'positions' (n_saddles, 2, N, 3), 'potential_energy', 'converged',
    'fmax' (n_saddles, 2)} and 'barriers' (n_saddles, 2), the saddle's energy minus each minimum's.  NumPy arrays or
    float64 CUDA tensors in, the same kind out."""

    def __init__(self, model, masses, n_saddles=1, E_to_eV=_KCAL_PER_MOL_IN_EV, F_to_eV_Ang=_KCAL_PER_MOL_IN_EV):
        self.n_saddles = int(n_saddles)
        if self.n_saddles < 1:
            raise ValueError('n_saddles must be >= 1')
        GDMLDynamics.__init__(self, model, masses, 2 * self.n_saddles, E_to_eV, F_to_eV_Ang)

    # ------------------------------------------------------------------ model units
    def _irc_raw(self, modes, max_points, step, fmax):
        """modes (n_saddles, 3N) -> (R_path (n_rep, max_points, 3N), E_path (n_rep, max_points), n_points, end, fmax
        (n_rep,)), in model units; step in the handle's mass-weighted unit."""
        if hasattr(modes, 'data_ptr'):  # the entry point copies n_saddles 3N doubles from this pointer
            _check_cuda_f64(modes, 'modes')
            modes = modes.contiguous()
        else:
            modes = np.ascontiguousarray(modes, dtype=np.float64)
        if tuple(modes.shape) != (self.n_saddles, 3 * self.n_atoms):
            raise ValueError('modes must be (n_saddles, 3N) = (%d, %d): %s' % (self.n_saddles, 3 * self.n_atoms,
                                                                                tuple(modes.shape)))
        n, mp = self.n_replicas, int(max_points)
        out = (self._empty((n, max(mp, 0), 3 * self.n_atoms)), self._empty((n, max(mp, 0))), self._empty(n, np.int64),
               self._empty(n, np.int32), self._empty(n))
        _lib.check(
            _lib.lib().sgdml_b200_irc_rk4(self._handle, _lib.ptr(modes), mp, float(step), float(fmax),
                                          *(_lib.ptr(x) for x in out), _lib.current_stream()),
            'irc_rk4',
        )
        return out

    # ------------------------------------------------------------------ ASE units
    def run(self, saddles, modes, step=0.05, max_points=500, fmax=0.05, relax_ends=True, relax_steps=1000):
        # both are checked before the state changes
        R = _per_unit(saddles, 'saddles', self.n_saddles, self.n_atoms, 'n_saddles')
        modes = _per_unit(modes, 'modes', self.n_saddles, self.n_atoms, 'n_saddles')
        if not (math.isfinite(float(step)) and float(step) > 0.0):
            raise ValueError('step must be finite and > 0')
        R = R.repeat_interleave(2, 0) if hasattr(R, 'data_ptr') else np.repeat(R, 2, axis=0)
        self.set_state(R.reshape(self.n_replicas, self.n_atoms, 3))
        # x = R / sqrt(inv_mass): amu^1/2 Angstrom -> the handle's unit (model length over sqrt of its inverse mass)
        c = self.F_to_eV_Ang * self.Ang_to_R * FS**2
        Rp, Ep, n_points, end, fm = self._irc_raw(modes, max_points, float(step) * self.Ang_to_R / math.sqrt(c),
                                                  float(fmax) / self.F_to_eV_Ang)
        g, mp = (self.n_saddles, 2), int(max_points)
        k = np.arange(mp, dtype=np.float64)[None, None, :]
        npt = _host(n_points).reshape(g + (1,))
        s = np.where(k < npt, np.array([1.0, -1.0])[None, :, None] * k * float(step), np.nan)
        if hasattr(Ep, 'data_ptr'):
            import torch

            s = torch.from_numpy(s).to(Ep.device)
        out = {'positions': (Rp / self.Ang_to_R).reshape(g + (mp, self.n_atoms, 3)),
               'energies': (Ep * self.E_to_eV).reshape(g + (mp,)), 's': s, 'n_points': n_points.reshape(g),
               'end': end.reshape(g), 'fmax': (fm * self.F_to_eV_Ang).reshape(g)}
        if relax_ends:
            m = self.relax(fmax=fmax, max_steps=relax_steps)
            E_min = m['potential_energy'].reshape(g)
            out['minima'] = {'positions': m['positions'].reshape(g + (self.n_atoms, 3)), 'potential_energy': E_min,
                             'converged': m['converged'].reshape(g), 'fmax': m['fmax'].reshape(g)}
            out['barriers'] = out['energies'][:, :, 0] - E_min
        return out


def _per_unit(x, name, n, N, what):
    """(n, N, 3) or (N, 3) -> (n, 3N), the same kind; torch inputs must be float64 CUDA tensors.  what: n's name."""
    if hasattr(x, 'data_ptr'):
        _check_cuda_f64(x, name)
    else:
        x = np.asarray(x)
    shape = tuple(x.shape)
    if shape == (N, 3):
        x = x.reshape(1, N, 3)
        x = x.expand(n, N, 3) if hasattr(x, 'data_ptr') else np.broadcast_to(x, (n, N, 3))
    elif shape != (n, N, 3):
        raise ValueError('%s must be (%s, N, 3) = (%d, %d, 3) or (N, 3): %s' % (name, what, n, N, shape))
    if hasattr(x, 'data_ptr'):
        return x.reshape(n, 3 * N).contiguous()
    return np.ascontiguousarray(x, dtype=np.float64).reshape(n, 3 * N)


def _check_cuda_f64(x, name):
    """A torch input handed to the engine as a pointer must be a float64 CUDA tensor."""
    import torch

    if x.dtype != torch.float64 or not x.is_cuda:
        raise ValueError('%s: torch inputs must be float64 CUDA tensors' % name)


def kabsch_align(x, ref):
    """x (..., N, 3) moved by the proper rotation and translation that minimise its squared distance to ref (Kabsch,
    Acta Cryst. A32, 922 (1976))."""
    x = np.asarray(x, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    cx = x.mean(-2, keepdims=True)
    cr = ref.mean(-2, keepdims=True)
    H = np.swapaxes(x - cx, -1, -2) @ (ref - cr)  # (..., 3, 3)
    U, _, Vt = np.linalg.svd(H)
    d = np.sign(np.linalg.det(np.swapaxes(Vt, -1, -2) @ np.swapaxes(U, -1, -2)))
    D = np.zeros(H.shape)
    D[..., 0, 0] = 1.0
    D[..., 1, 1] = 1.0
    D[..., 2, 2] = np.where(d == 0.0, 1.0, d)
    rot = U @ D @ Vt  # row vectors: x_aligned = (x - cx) rot + cr
    return (x - cx) @ rot + cr
