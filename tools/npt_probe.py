"""Steps per second of GDMLNPTDynamics on the device against NVT GDMLDynamics at the same replica count, and against the
host loop it replaces.

For the ethanol and aspirin synthetic models (synth.random_model on the benchmark's shapes) made periodic with a cubic
cell of 20 L (a dense-enough box that the minimum-image convention is exercised, and the same cell for every run):
  npt:  GDMLNPTDynamics.run, 300 K, friction 0.01 / fs, 1 bar-scale target pressure, compressibility 0.01 A^3/eV,
        tau_p 100 fs, no frames: one step graph of k_npt_step and the forces with the virial in per-replica cells
  nvt:  GDMLDynamics.run with the same replica count, temperature and friction (k_md_step and the plain forces in the
        model's cell)
  host: at B = 1, the ASE-shaped route: GDMLPredict.predict_virial on NumPy positions with one cell per geometry, plus
        a NumPy BAOAB and barostat step (one predict call and one host round trip per step)
B = 1, 16, 256 and 4096 replicas.  Wall clock around runs that end in a device synchronise, after a warm-up run; each
rate is the median of `--reps` timed windows of about `--window` seconds.  Prints JSON with the card's name, power
limit and max SM clock read in the same run; `--out FILE` also writes it to FILE."""

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
from md_probe import _gpu_info, _rate  # noqa: E402


def _host_loop(gp, R, lat, s, dt, gamma, kT, P0, beta_T, tau_p):
    """One replica's host route: predict_virial in its cell, then the BAOAB and barostat step in NumPy."""
    rng = np.random.default_rng(0)
    st = {'R': R.copy(), 'V': np.zeros_like(R), 'L': lat.copy()}
    E, F, W = gp.predict_virial(st['R'], lattice=st['L'][None])
    st['F'], st['W'] = F, W
    h, c1 = 0.5 * dt, np.exp(-gamma * dt)
    sig = np.sqrt((1.0 - c1 * c1) * kT * s)
    c_a, c_b = beta_T / tau_p * dt, 2.0 * kT * beta_T / tau_p * dt

    def run(n):
        for _ in range(n):
            V, R, L, F, W = st['V'], st['R'], st['L'], st['F'], st['W']
            vol = abs(np.linalg.det(L))
            pint = ((V * V / s).sum() + np.trace(W[0])) / (3.0 * vol)
            de = -c_a * (P0 - pint) + np.sqrt(c_b / vol) * rng.standard_normal()
            mu = np.exp(de / 3.0)
            V = V + h * (F * s)
            R = R + h * V
            V = c1 * V + sig * rng.standard_normal(V.shape)
            R = (R + h * V) * mu
            V = V / mu
            L = L * mu
            _, F, W = gp.predict_virial(R, lattice=L[None])
            st.update(R=R, V=V + h * (F * s), L=L, F=F, W=W)

    return run


def _workload(name, batches, window, reps):
    import torch

    import sgdml_b200
    from sgdml_b200 import md, synth

    cfg = synth.CONFIGS[name]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms, r0 = synth.config_perms_and_r0(name)
    model = synth.random_model(N, M, perms, cfg['sig'], r0=r0)
    model['lattice'] = 20.0 * np.eye(3)
    gp = sgdml_b200.GDMLPredict(model)
    masses = np.full(N, 12.0)
    dt, fric, T = 0.5, 0.01, 300.0
    p_au, comp_au, taup = 6.2e-7, 0.01, 100.0  # eV/A^3 (about 1 bar), A^3/eV, fs
    res = {'workload': name, 'N': N, 'M': M, 'S': int(perms.shape[0]), 'dt_fs': dt, 'cell_L': 20.0, 'rows': []}
    Rall = synth.geometries(N, max(batches), 1, r0=r0)
    for B in batches:
        row = {'B': B}
        npt = sgdml_b200.GDMLNPTDynamics(gp, masses, n_replicas=B)
        nvt = sgdml_b200.GDMLDynamics(gp, masses, n_replicas=B)
        npt.set_state(Rall[:B])
        nvt.set_state(Rall[:B])
        runs = {'npt': lambda n: npt.run(n, dt, T, fric, p_au, comp_au, taup),
                'nvt': lambda n: nvt.run(n, dt, temperature_K=T, friction_per_fs=fric)}
        for label, fn in runs.items():
            def step(n, fn=fn):
                fn(n)
                torch.cuda.synchronize()

            step(20)  # capture and warm-up
            sps, n = _rate(step, window, reps)
            row[label + '_steps_per_s'] = sps
            row[label + '_replica_steps_per_s'] = sps * B
            row[label + '_steps_per_window'] = n
        row['npt_over_nvt'] = row['npt_steps_per_s'] / row['nvt_steps_per_s']
        if B == 1:
            kc = npt.E_to_eV
            s = np.repeat(npt.inv_mass, 3)
            host = _host_loop(gp, Rall[:1].reshape(1, -1), model['lattice'], s, dt, fric, md.KB_EV * T / kc,
                              p_au / kc, comp_au * kc, taup)
            host(20)
            sps, n = _rate(host, window, reps)
            row['host_steps_per_s'] = sps
            row['npt_over_host'] = row['npt_steps_per_s'] / sps
        print(json.dumps(row), flush=True)
        res['rows'].append(row)
        del npt, nvt
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--window', type=float, default=0.3, help='seconds per timed window')
    ap.add_argument('--out', default=None, help='also write the JSON results to this file')
    a = ap.parse_args()
    from sgdml_b200 import _lib

    _lib.require_gpu()
    res = {'gpu': _gpu_info()}
    print(json.dumps(res), flush=True)
    for name in ('ethanol', 'aspirin'):
        res[name] = _workload(name, (1, 16, 256, 4096), a.window, a.reps)
    res['gpu_after'] = _gpu_info()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
