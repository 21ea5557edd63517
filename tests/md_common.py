"""Helpers shared by the device dynamics tests (test_md.py, test_pimd.py, test_relax.py, test_relax_oracle.py): the
model fixtures they run on, masses in model units, forces from the engine's predictor, and a harmonic spring surface
with its training task."""

import numpy as np
import pytest

FIXTURES_MD = ['n5_m10_s1', 'n9_m16_s6', 'n12_m8_s12', 'n21_m6_s6', 'ecstr_n6_m8', 'pbc_n6_m8', 'big_n100_m2_s12',
               'big_n240_m2_s3']


def md_fs_masses(m):
    """Masses (amu) for which GDMLDynamics with E_to_eV = F_to_eV_Ang = 1 has the inverse masses 1 / m (model units,
    femtoseconds)."""
    from sgdml_b200 import md

    return md.FS**2 * np.asarray(m, dtype=np.float64)


def _cuda_forces(gp):
    import torch

    def forces(R):
        E, F = gp.predict(torch.from_numpy(np.ascontiguousarray(R)).cuda())
        return E.cpu().numpy(), F.cpu().numpy()

    return forces


# harmonic pair springs about the base geometry: a bound PES with a clear minimum
_N_SPRING, _K_SPRING = 5, 2.0


def _spring_pes(R):
    from sgdml_b200 import synth

    r0 = synth.base_geometry(_N_SPRING)
    d0 = np.sqrt(((r0[:, None] - r0[None]) ** 2).sum(-1))
    R = np.asarray(R, dtype=np.float64).reshape(-1, _N_SPRING, 3)
    diff = R[:, :, None, :] - R[:, None, :, :]
    d = np.sqrt((diff * diff).sum(-1)) + np.eye(_N_SPRING)
    ext = (d - d0 - np.eye(_N_SPRING)) * (1 - np.eye(_N_SPRING))
    E = 0.25 * _K_SPRING * (ext * ext).sum((1, 2))
    F = -_K_SPRING * (ext[..., None] * diff / d[..., None]).sum(2)
    return E, F


def make_spring_task():
    from sgdml_b200 import synth

    task = synth.make_task(_N_SPRING, 60, np.arange(_N_SPRING)[None], 4, seed=3)
    task['E_train'], task['F_train'] = _spring_pes(task['R_train'])
    task['dataset_theory'] = 'harmonic_springs'
    return task


@pytest.fixture(scope='module')
def spring_task():
    return make_spring_task()
