"""Generates tests/golden/big_n240_m2_s3.npz and big_n370_m2_s3.npz by running the UNMODIFIED reference
(stefanch/sGDML v1.0.3) on seeded synthetic molecules with hundreds of atoms: beyond the predictor's shared-memory
finishing kernel (N >= 227) and the old 128-atom bound of the energy-constraint kernels.  Run in the build container
only (the reference is not on the GPU box):

    cp -r /root/reference/sgdml baseline/_ref/          # writable copy (predict.py:1046-1074)
    PYTHONPATH=baseline/_ref:. python tests/golden/make_golden_big.py

Each fixture holds, for a synthetic N-atom molecule with M = 2 and S = 3 (one rotor): a few columns of K
(index-list mode), the M energy-constraint columns (use_E_cstr) and the predictions of a random-coefficient model on
query geometries; at N = 240 also those of the same model with random alphas_E.  The arrays of length D (descriptors,
their Jacobians, R_d_desc_alpha, the rows of tril_perms_lin) are kept at every DESC_STRIDE-th descriptor entry only, so
that each file stays small: the tests recompute them and compare there.
"""

import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, 'baseline', '_ref'))

_spec = importlib.util.spec_from_file_location('synth', os.path.join(ROOT, 'sgdml_b200', 'synth.py'))
synth = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(synth)

import sgdml  # noqa: E402  (the reference)
from sgdml.predict import GDMLPredict  # noqa: E402
from sgdml.train import GDMLTrain  # noqa: E402
from sgdml.utils.desc import Desc  # noqa: E402

assert sgdml.__version__ == '1.0.3'

DESC_STRIDE = 53
N_COLS = 4


def make(gdml_train, N):
    M, sig = 2, 50
    perms = synth.rotor_swap_group(N, 1, 0)
    S = len(perms)
    task = synth.make_task(N, M, perms, sig)
    desc = Desc(N, max_processes=1)
    tril_perms = np.array([Desc.perm(p) for p in perms])
    tril_perms_lin = (tril_perms + np.arange(S)[:, None] * desc.dim).flatten('F')
    R = task['R_train'].reshape(M, -1)
    R_desc, R_d_desc = desc.from_R(R, max_processes=1)
    cols = np.arange(3 * N, 6 * N, 3 * N // N_COLS)
    K_cols = gdml_train._assemble_kernel_mat(R_desc, R_d_desc, tril_perms_lin, sig, desc, col_idxs=cols)
    ecols = np.arange(3 * N * M, 3 * N * M + M)
    K_ecols = gdml_train._assemble_kernel_mat(R_desc, R_d_desc, tril_perms_lin, sig, desc, use_E_cstr=True, col_idxs=ecols)
    rng = np.random.default_rng(N)
    alphas_F = rng.standard_normal(M * 3 * N)
    alphas_E = rng.standard_normal(M)
    model = gdml_train.create_model(task, 'analytic', R_desc, R_d_desc, tril_perms_lin, 0.6, alphas_F)
    model['c'] = 12.5
    R_query = synth.geometries(N, 2, 1).reshape(2, -1)
    E_q, F_q = GDMLPredict(model, max_processes=1, use_torch=False).predict(R_query)
    extra = {}
    if N == 240:
        task_e = dict(task, use_E_cstr=True)
        model_e = gdml_train.create_model(task_e, 'analytic', R_desc, R_d_desc, tril_perms_lin, 0.6, alphas_F, alphas_E)
        model_e['c'] = 12.5
        extra['E_query_ecstr'], extra['F_query_ecstr'] = GDMLPredict(model_e, max_processes=1, use_torch=False).predict(R_query)
        extra['alphas_E'] = alphas_E
    idx = np.arange(0, desc.dim, DESC_STRIDE)
    name = 'big_n%d_m%d_s%d' % (N, M, S)
    out = os.path.join(HERE, name + '.npz')
    np.savez_compressed(
        out,
        reference_version=sgdml.__version__,
        n_atoms=N,
        perms=perms,
        sig=sig,
        lam=task['lam'],
        z=task['z'],
        R_train=task['R_train'],
        desc_idx=idx,
        tril_perms_lin_sub=tril_perms_lin.astype(np.int64).reshape(desc.dim, S)[idx],
        R_desc_sub=R_desc[:, idx],
        R_d_desc_sub=R_d_desc[:, idx],
        K_cols=K_cols,
        cols=cols,
        K_ecols=K_ecols,
        ecols=ecols,
        alphas_F=alphas_F,
        R_d_desc_alpha_sub=model['R_d_desc_alpha'][:, idx],
        std=model['std'],
        c=model['c'],
        R_query=R_query,
        E_query=E_q,
        F_query=F_q,
        **extra,
    )
    print(name + ': K_cols', K_cols.shape, 'K_ecols', K_ecols.shape, 'size %.0f KB' % (os.path.getsize(out) / 1024))


if __name__ == '__main__':
    gdml_train = GDMLTrain(max_processes=1, use_torch=False)  # one instance per process (train.py:336-342)
    for n_atoms in (240, 370):
        make(gdml_train, n_atoms)
