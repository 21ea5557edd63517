"""B = 1 latency of the predictor from host NumPy buffers (the MD stepping path): CUDA-graph replay with zero-copy host
buffers, graph replay with copy nodes, plain launches."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import sgdml_b200
from sgdml_b200 import synth
shapes = [('aspirin', None), ('ethanol', None)]
# one synthetic molecule per further tile configuration: DP = 72 (N = 12), 112 (N = 15), 160 (N = 18)
shapes += [('N%d' % N_, dict(n_atoms=N_, n_train=1000, n_rotors=1, n_swaps=1, sig=20)) for N_ in (12, 15, 18)]
if os.environ.get('LATENCY_SHAPES'):
    shapes = [s_ for s_ in shapes if s_[0] in os.environ['LATENCY_SHAPES'].split(',')]
for wl, cfg in shapes:
    cfg = cfg or synth.CONFIGS[wl]
    N, M = cfg['n_atoms'], cfg['n_train']
    perms = synth.rotor_swap_group(N, cfg['n_rotors'], cfg['n_swaps'])
    model = synth.random_model(N, M, perms, cfg['sig'])
    R1 = synth.geometries(N, 1, 1).reshape(1, -1)
    for name, env in (('graph replay, zero-copy', {'SGDML_B200_GRAPH': '1', 'SGDML_B200_GRAPH_ZEROCOPY': '1'}),
                      ('graph replay, copy nodes', {'SGDML_B200_GRAPH': '1', 'SGDML_B200_GRAPH_ZEROCOPY': '0'}),
                      ('plain launches', {'SGDML_B200_GRAPH': '0'})):
        os.environ.update(env)
        p1 = sgdml_b200.GDMLPredict(model)  # a fresh handle: the graph cache is per model
        for _ in range(20): p1.predict(R1)
        t0 = time.perf_counter()
        for _ in range(1000): p1.predict(R1)
        print('%s B=1 host NumPy in/out, %s: %.1f us per call' % (wl, name, (time.perf_counter() - t0) / 1000 * 1e6), flush=True)
    os.environ.pop('SGDML_B200_GRAPH', None)
    os.environ.pop('SGDML_B200_GRAPH_ZEROCOPY', None)
