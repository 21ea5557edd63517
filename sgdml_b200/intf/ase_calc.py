"""ASE calculator on the H100 engine -- the reference's ``sgdml.intf.ase_calc.SGDMLCalculator``
(intf/ase_calc.py:36-110): same constructor arguments, unit handling and ``results`` layout, float64 end to end
(the reference's torch path downcasts positions to float32, predict.py:1197-1201).

MD drivers call ``calculate`` with ONE geometry at a time: that call goes through the engine's small-batch path
(sweep over the training points split across CTAs, the launch sequence replayed from a CUDA graph,
``sgdml_b200_predict`` in csrc/predict.cu).

ASE itself is optional (as in the reference, which raises ImportError without it): ``SGDMLCalculatorCore`` holds
everything that does not need ASE and is what the tests exercise; ``SGDMLCalculator`` exists only when ASE imports.
"""

import logging

import numpy as np

from ..predict import GDMLPredict

# ase.units: kcal / mol in eV (CODATA 2014 values as ASE uses them): 4.184e3 J / (N_A e)
_KCAL_PER_MOL_IN_EV = 4.184e3 / (6.022140857e23 * 1.6021766208e-19)


class SGDMLCalculatorCore(object):
    """Unit conversion + prediction of intf/ase_calc.py:81-110, without the ASE base class.  Periodic models also
    implement 'stress' (an extension: the reference has none), from the engine's virial W = -dE/d(eps):
    sigma = -W E_to_eV / V in eV/A^3, Voigt order (xx, yy, zz, yz, xz, xy).

    use_atoms_cell=False (default): E, F and stress in the model's own cell, whatever cell the atoms carry.
    use_atoms_cell=True: every call evaluates the model in the cell it is given (ASE's atoms.cell, vectors as ROWS in
    Angstrom, becomes cell^T * Ang_to_R in the model's column convention) -- what NPT dynamics and variable-cell
    relaxations need.  Only periodic models have a cell to replace."""

    implemented_properties = ['energy', 'forces']

    def _setup(self, model_path, E_to_eV, F_to_eV_Ang, use_torch=False, use_atoms_cell=False):
        self.log = logging.getLogger(__name__)
        model = model_path if isinstance(model_path, dict) else np.load(model_path, allow_pickle=True)
        self.gdml_predict = GDMLPredict(model, use_torch=use_torch)
        self.periodic = self.gdml_predict.lat_and_inv is not None
        if use_atoms_cell and not self.periodic:
            raise ValueError('use_atoms_cell needs a periodic model (one with a lattice): this model has no cell to replace')
        self.use_atoms_cell = bool(use_atoms_cell)
        self.implemented_properties = ['energy', 'forces'] + (['stress'] if self.periodic else [])
        self.gdml_predict.prepare_parallel(n_bulk=1)  # ase_calc.py:84 (a no-op tuning call on the engine)
        self.log.warning(
            "Please remember to specify the proper conversion factors, if your model does not use 'kcal/mol' and 'Ang' as units."
        )
        self.E_to_eV = E_to_eV  # energy unit of the model -> eV
        self.Ang_to_R = F_to_eV_Ang / E_to_eV  # Angstrom -> length unit of the model (ase_calc.py:93-94)
        self.F_to_eV_Ang = F_to_eV_Ang  # force unit of the model -> eV/Ang

    def compute(self, positions, cell=None, stress=False):
        """positions (N, 3) in Angstrom -> {'energy': eV, 'forces': (N, 3) eV/Ang} (ase_calc.py:98-110).
        cell: (3, 3) cell in Angstrom with the lattice vectors as ROWS (ASE's atoms.cell) to evaluate a periodic model
        in for this call; None: the model's own cell.  stress=True adds 'stress' (6,) in eV/A^3, Voigt order."""
        r = np.array(positions, dtype=np.float64) * self.Ang_to_R
        if (stress or cell is not None) and not self.periodic:
            raise ValueError('stress and per-call cells need a periodic model (one with a lattice); this model is a '
                             'free molecule')
        if not stress and cell is None:
            e, f = self.gdml_predict.predict(r.ravel())
            e = e * self.E_to_eV
            f = f * self.F_to_eV_Ang
            return {'energy': e, 'forces': f.reshape(-1, 3)}
        lat = None if cell is None else np.ascontiguousarray(np.asarray(cell, dtype=np.float64).T * self.Ang_to_R)
        e, f, w = self.gdml_predict.predict_virial(r.ravel(), lattice=lat)
        out = {'energy': e * self.E_to_eV, 'forces': (f * self.F_to_eV_Ang).reshape(-1, 3)}
        if stress:
            cell_ang = np.asarray(cell, dtype=np.float64) if cell is not None else self.gdml_predict.lat_and_inv[0] / self.Ang_to_R
            vol = abs(np.linalg.det(cell_ang))
            s = -w[0] * self.E_to_eV / vol
            out['stress'] = np.array([s[0, 0], s[1, 1], s[2, 2], s[1, 2], s[0, 2], s[0, 1]])
        return out


try:
    from ase.calculators.calculator import Calculator
    from ase.units import kcal, mol

    class SGDMLCalculator(Calculator, SGDMLCalculatorCore):
        implemented_properties = ['energy', 'forces']

        def __init__(self, model_path, E_to_eV=kcal / mol, F_to_eV_Ang=kcal / mol, use_torch=False,
                     use_atoms_cell=False, *args, **kwargs):
            super(SGDMLCalculator, self).__init__(*args, **kwargs)
            self._setup(model_path, E_to_eV, F_to_eV_Ang, use_torch=use_torch, use_atoms_cell=use_atoms_cell)

        def calculate(self, atoms=None, properties=('energy',), *args, **kwargs):
            super(SGDMLCalculator, self).calculate(atoms, properties, *args, **kwargs)
            cell = np.asarray(self.atoms.cell) if self.use_atoms_cell else None
            self.results = self.compute(self.atoms.get_positions(), cell=cell, stress='stress' in properties)

except ImportError:

    def __getattr__(name):
        if name == 'SGDMLCalculator':
            raise ImportError("Optional ASE dependency not found! Please run 'pip install sgdml[ase]' to install it.")
        raise AttributeError(name)
