"""Where the aspirin prediction step goes outside the main kernel's tile loop.

    python tools/predict_overhead_probe.py [B]

Prints the card and its power limit, then for the aspirin workload (bench config 2, random-coefficient model, device
resident queries, B = 65 536 by default):
  * the step time (CUDA events, profiler off) and the device time per step of each profiled kernel family
    (desc, predict_aux, predict_main, predict_finish);
  * the main kernel at M = 1000 and M = 2000 training points.  Its time is linear in M, so the intercept 2 t(1000) -
    t(2000) is the cost per step that does not scale with the sweep over M: filling and draining the CTAs, the Q tiles,
    the G stores.  Divided by the CTAs that ran one after another on each SM it gives the fixed cost per query tile."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import sgdml_b200  # noqa: E402
from sgdml_b200 import _lib, synth  # noqa: E402

FAMILIES = ('desc', 'predict_aux', 'predict_main', 'predict_finish')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = torch.cuda.get_device_name(0) + ', power limit unknown'
    return q


def step_ms(p, R, reps=10):
    for _ in range(3):
        p.predict(R)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        p.predict(R)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def families_ms(p, R, reps=5):
    L = _lib.lib()
    L.sgdml_b200_profile_reset()
    L.sgdml_b200_profile_enable(1)
    for _ in range(reps):
        p.predict(R)
    torch.cuda.synchronize()
    L.sgdml_b200_profile_enable(0)
    snap = _lib.profile_snapshot()
    return {f: snap[f][0] / reps for f in FAMILIES}


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
    print('card:', card())
    cfg = synth.CONFIGS['aspirin']
    N = cfg['n_atoms']
    perms, r0 = synth.config_perms_and_r0('aspirin')
    S = len(perms)
    R = torch.from_numpy(synth.geometries(N, B, 1, r0=r0).reshape(B, -1)).cuda()
    main_ms = {}
    for M in (1000, 2000):
        p = sgdml_b200.GDMLPredict(synth.random_model(N, M, perms, cfg['sig'], r0=r0))
        t = step_ms(p, R)
        fam = families_ms(p, R)
        main_ms[M] = fam['predict_main']
        print('M %d  B %d  S %d  step %.3f ms  ' % (M, B, S, t)
              + '  '.join('%s %.3f ms' % (f, fam[f]) for f in FAMILIES)
              + '  outside main %.3f ms (%.1f %%)' % (t - fam['predict_main'], 100 * (t - fam['predict_main']) / t))
        if M == 1000:
            t1000, fam1000 = t, fam
        del p
    icpt = 2 * main_ms[1000] - main_ms[2000]
    # query tiles per step (BQ 32 rows at D = 210) and the CTAs that ran one after another on each SM
    tiles = B * S / 32.0
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    waves = tiles / sms
    print('main kernel intercept %.3f ms per step; %.0f query tiles on %d SMs = %.1f per SM: %.2f us per tile'
          % (icpt, tiles, sms, waves, 1e3 * icpt / waves))
    share = (fam1000['predict_aux'] + max(icpt, 0.0)) / t1000
    print('predict_aux + intercept = %.3f ms = %.2f %% of the step' % (fam1000['predict_aux'] + max(icpt, 0.0), 100 * share))


if __name__ == '__main__':
    main()
