"""Times GDMLTrain.train with the iterative solver (Nystroem-preconditioned CG) on a named synthetic
config at a chosen number of training points; runs on 1 GPU or under torchrun (one rank per GPU:
row-sharded K.v and Nystroem factor)."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, __file__.rsplit('/', 2)[0])
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--workload', default='ac-ala3-nhme')
ap.add_argument('--n-train', type=int, default=500)
ap.add_argument('--max-memory', type=float, default=8.0, help='GB; below the analytic estimate -> CG')
ap.add_argument('--n-query', type=int, default=64)
ap.add_argument('--profile', action='store_true', help='per-kernel-family device times (adds synchronisation)')
ap.add_argument('--trace', type=int, default=0, help='print the CG residual every this many iterations')
ap.add_argument('--E-cstr', action='store_true', help='energy constraints in the kernel: the (3NM + M)-square system')
a = ap.parse_args()

world = int(os.environ.get('WORLD_SIZE', '1'))
rank = int(os.environ.get('RANK', '0'))
if world > 1:
    import torch.distributed as dist

    os.environ.setdefault('NCCL_DEBUG', 'WARN')
    torch.cuda.set_device(int(os.environ.get('LOCAL_RANK', '0')))
    dist.init_process_group('nccl', device_id=torch.device('cuda', torch.cuda.current_device()))

import sgdml_b200  # noqa: E402
from sgdml_b200 import synth  # noqa: E402

task = synth.make_config_task(a.workload, n_train=a.n_train)
task['use_E_cstr'] = a.E_cstr
N = task['R_train'].shape[1]
np.random.seed(0)
trainer = sgdml_b200.GDMLTrain(max_memory=a.max_memory)
trainer.distributed = world > 1  # every rank runs this script: the iterative solver shards over them
torch.cuda.synchronize()
t0 = time.perf_counter()
_n_cb = [0]


def _cb(*args, **kw):
    if 'sec_disp_str' in kw and 'iter' in str(kw.get('sec_disp_str')):
        _n_cb[0] += 1
        if a.trace and rank == 0 and _n_cb[0] % a.trace == 0:
            print('[%.1fs] %s | %s' % (time.perf_counter() - t0, kw.get('disp_str'), kw.get('sec_disp_str')), file=sys.stderr, flush=True)


from sgdml_b200 import _lib  # noqa: E402

if a.profile:
    _lib.lib().sgdml_b200_profile_reset()
    _lib.lib().sgdml_b200_profile_enable(1)
model = trainer.train(task, callback=_cb if a.trace else None)
if a.profile:
    _lib.lib().sgdml_b200_profile_enable(0)
    if rank == 0:
        print('profile (ms, scopes, launches):', {k: (round(v[0], 1), v[1], v[2]) for k, v in _lib.profile_snapshot().items()}, file=sys.stderr)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
_, r0 = synth.config_perms_and_r0(a.workload)
Rq = synth.geometries(N, a.n_query, 1, r0=r0)
_, Fq = synth.toy_pes(Rq)
_, F = sgdml_b200.GDMLPredict(model).predict(Rq.reshape(a.n_query, -1))
err = float(np.sqrt(np.mean((F - Fq.reshape(a.n_query, -1)) ** 2)) / np.sqrt(np.mean(Fq**2)))
if rank == 0:
    out = {
        'workload': a.workload,
        'n_gpus': world,
        'n_atoms': N,
        'n_train': a.n_train,
        'n_perms': int(len(task['perms'])),
        'use_E_cstr': bool(a.E_cstr),
        'n': 3 * N * a.n_train + (a.n_train if a.E_cstr else 0),
        'solver': str(model['solver_name']),
        'train_s': dt,
        'timings': {k: float(v) for k, v in trainer.timings.items()},
        'force_rmse_rel_heldout': err,
    }
    if 'solver_iters' in model:
        out.update(
            iters=int(model['solver_iters']),
            n_inducing_cols=int(len(model['inducing_pts_idxs'])),
            resid_rel=float(model['solver_resid'] / model['norm_y_train']),
            setup_s=float(trainer.timings.get('precon_s', float('nan'))),  # leverage scores + preconditioner
            cg_s_per_iter=float(trainer.timings['cg_s'] / max(1, trainer.timings['iters'])),
        )
    print(json.dumps(out))
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
