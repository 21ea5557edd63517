"""Generates tests/golden/cg_ecstr_n9_m40.npz by running the UNMODIFIED reference (stefanch/sGDML v1.0.3) on the
seeded synthetic task of make_golden.py's `iterative` fixture, with energy constraints in the kernel (use_E_cstr).
Run in the build container only (the reference is not on the GPU box):

    cp -r /root/reference/sgdml baseline/_ref/          # writable copy (predict.py:1046-1074)
    PYTHONPATH=baseline/_ref:. python tests/golden/make_golden_cg_ecstr.py

The system is (3NM + M)-square in the layout [forces; energies] (train.py:939-947), inducing columns are drawn from
all 3NM + M columns and may be energy columns (iterative.py:372-379), the operator returns [F; -E]
(iterative.py:183-204) and the model carries alphas_E (iterative.py:685-698, train.py:1052-1056).  The fixture holds
the inputs, the reference's inducing columns, coefficients, solver keys, leverage scores, P.v for a fixed v, its K_nm
at the inducing columns and its predictions on query geometries.
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
from sgdml.solvers.iterative import Iterative  # noqa: E402
from sgdml.train import GDMLTrain  # noqa: E402
from sgdml.utils.desc import Desc  # noqa: E402

assert sgdml.__version__ == '1.0.3'


def main():
    N, M, sig = 9, 40, 20
    perms = synth.rotor_swap_group(N, 1, 1)
    task = synth.make_task(N, M, perms, sig)
    task['use_E_cstr'] = True
    n_F = 3 * N * M
    max_memory = 0.004  # GB -> a handful of inducing points (iterative.py:826-843)
    gdml_train = GDMLTrain(max_memory=max_memory, max_processes=1, use_torch=False)
    np.random.seed(1234)
    model = gdml_train.train(task)
    assert model['solver_name'] == 'cg'
    idxs = np.asarray(model['inducing_pts_idxs'])
    assert np.any(idxs >= n_F), 'the seed must draw at least one energy column'
    desc = Desc(N, max_processes=1)
    R = task['R_train'].reshape(M, -1)
    R_desc, R_d_desc = desc.from_R(R, max_processes=1)
    lin = model['tril_perms_lin']

    it = Iterative(gdml_train, desc, max_memory, 1, False)
    P_op, lev_scores = it._init_precon_operator(task, R_desc, R_d_desc, lin, idxs)
    rng = np.random.default_rng(7)
    v = rng.standard_normal(n_F + M)
    P_op @ v  # first call only "primes" the operator (iterative.py:122-125)
    Pv = P_op @ v
    K_nm = gdml_train._assemble_kernel_mat(R_desc, R_d_desc, lin, sig, desc, use_E_cstr=True, col_idxs=idxs)
    # the run above may restart with more inducing columns when CG stalls (iterative.py:726-801), and solver_iters
    # counts the iterations of every attempt: solve again with the final columns (reused, iterative.py:518-520) for
    # the iteration count of one CG run on them
    fixed = gdml_train.train(dict(task, inducing_pts_idxs=idxs))
    assert np.array_equal(fixed['inducing_pts_idxs'], idxs)

    predictor = GDMLPredict(model, max_processes=1, use_torch=False)
    R_query = synth.geometries(N, 10, 1).reshape(10, -1)
    E_q, F_q = predictor.predict(R_query)
    E_train = task['E_train'].ravel()
    y = np.hstack((task['F_train'].ravel(), -E_train + np.mean(E_train))) / model['std']  # train.py:939-947
    out = os.path.join(HERE, 'cg_ecstr_n9_m40.npz')
    np.savez_compressed(
        out,
        reference_version=sgdml.__version__,
        n_atoms=N,
        n_train=M,
        perms=perms,
        sig=sig,
        lam=task['lam'],
        max_memory_gb=max_memory,
        inducing_pts_idxs=idxs,
        alphas_F=model['alphas_F'],
        alphas_E=model['alphas_E'],
        solver_iters=model['solver_iters'],
        solver_iters_fixed_cols=fixed['solver_iters'],
        solver_resid=model['solver_resid'],
        solver_tol=model['solver_tol'],
        norm_y_train=model['norm_y_train'],
        std=model['std'],
        c=model['c'],
        lev_scores=lev_scores,
        v=v,
        Pv=Pv,
        K_nm=K_nm,
        R_query=R_query,
        E_query=E_q,
        F_query=F_q,
        y=y,
    )
    print(
        'cg_ecstr_n9_m40: %d inducing columns (%d energy columns), %d iterations (%d on the final columns), resid %.3e '
        '(tol*|y| = %.3e), size %.0f KB'
        % (len(idxs), int(np.sum(idxs >= n_F)), model['solver_iters'], fixed['solver_iters'], model['solver_resid'],
           model['solver_tol'] * model['norm_y_train'], os.path.getsize(out) / 1024)
    )


if __name__ == '__main__':
    main()
