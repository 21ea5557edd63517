"""Device time of GDMLPosterior: the factorisation, and per query the cross-row assembly, the TRSM against the factor
and k_posterior_blocks.

Models trained on the device from synthetic tasks at the ethanol (N = 9, M = 200, S = 6) and aspirin (N = 21,
M = 1000, S = 6) shapes of synth.CONFIGS.  For B = 1, 64 and 1024 query geometries the three stages of every chunk are
bracketed with CUDA events (one warm-up call first); the TRSM's achieved FP64 rate n^2 d B / t stands next to the
Cholesky's n^3 / 3 / t.  Prints JSON with the card's name and power limit read in the same run; `--out FILE` also
writes it to FILE."""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def _gpu_info():
    return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                    '--format=csv,noheader'], text=True).strip()


def _stages(post, R):
    """Device ms of (assembly, TRSM, blocks) over the chunks of one predict_cov(R)."""
    import torch

    from sgdml_b200 import _lib

    L = _lib.lib()
    B, n = R.shape[0], post.n
    c = post._chunk(B)
    ms = np.zeros(3)
    out = np.empty((B, post.dim, post.dim))
    for b0 in range(0, B, c):
        b1 = min(b0 + c, B)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        V, P = post._cross_rows(np.ascontiguousarray(R[b0:b1]))
        ev[1].record()
        _lib.check(L.sgdml_b200_trsm_right_lt(post._L.data_ptr(), n, post.ldl, V.data_ptr(), V.shape[0], V.shape[1],
                                              _lib.current_stream()), 'trsm_right_lt')
        ev[2].record()
        _lib.check(L.sgdml_b200_posterior_blocks(V.data_ptr(), V.shape[1], n, b1 - b0, post.n_atoms, P.data_ptr(),
                                                 post.scale, _lib.ptr(out[b0:b1]), _lib.current_stream()),
                   'posterior_blocks')
        ev[3].record()
        torch.cuda.synchronize()
        ms += [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]
        del V, P
    return ms, c


def run(configs, batches):
    import torch

    import sgdml_b200
    from sgdml_b200 import synth

    res = {'gpu': _gpu_info(), 'configs': {}}
    for name in configs:
        cfg = synth.CONFIGS[name]
        task = synth.make_config_task(name)
        gt = sgdml_b200.GDMLTrain()
        model = gt.train(task)
        gt.release_buffers()
        post = sgdml_b200.GDMLPosterior(model, task)
        n, d = post.n, post.dim
        t = post.timings
        entry = {'N': cfg['n_atoms'], 'M': cfg['n_train'], 'n': n, 'd': d,
                 'assemble_K_s': t['assemble_s'], 'factor_s': t['factor_s'],
                 'cholesky_tflops': n ** 3 / 3 / t['factor_s'] * 1e-12, 'batches': {}}
        perms, r0 = synth.config_perms_and_r0(name)
        for B in batches:
            R = synth.geometries(cfg['n_atoms'], B, 1, r0=r0).reshape(B, -1)
            _stages(post, R[:1])  # warm-up
            ms, c = _stages(post, R)
            entry['batches'][B] = {
                'chunk': c, 'assembly_ms_per_query': ms[0] / B, 'trsm_ms_per_query': ms[1] / B,
                'blocks_ms_per_query': ms[2] / B, 'total_ms_per_query': ms.sum() / B,
                'trsm_tflops': n * n * d * B / (ms[1] * 1e-3) * 1e-12}
            print(name, B, json.dumps(entry['batches'][B]), flush=True)
        res['configs'][name] = entry
        post.release()
        del post, model
        torch.cuda.empty_cache()
    res['gpu_after'] = _gpu_info()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='ethanol,aspirin')
    ap.add_argument('--batches', default='1,64,1024')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    res = run(a.configs.split(','), [int(b) for b in a.batches.split(',')])
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s)


if __name__ == '__main__':
    main()
