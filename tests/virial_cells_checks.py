"""Helpers for virials with one cell per geometry (sgdml_b200_predict_virial_cells, dist.predict_virial_sharded,
TrainPointShardedPredictor.predict_virial): seeded per-geometry cells, the oracle evaluated in each geometry's own cell,
and the componentwise checks of predict_checks / virial_checks applied row by row.  Plain functions on NumPy arrays,
shared by the CPU (gloo) and GPU tests."""

import numpy as np

import predict_checks as pc
import virial_checks as vc
from oracle import predict as opredict


def cells_for(R, base, seed, rows=None, spread=0.08):
    """(B, 3, 3) cells, one per geometry of R (B, 3N): `base` (lattice vectors as columns) scaled by 1 +- spread per
    axis and sheared by up to spread, drawn per geometry.  For the geometries in `rows` (default: all) a cell is
    redrawn until no pair of that geometry lies within 1e-6 of a rounding tie (pc.pbc_margin), so that the engine and
    the oracle pick the same image."""
    R = np.asarray(R, dtype=np.float64)
    B = R.shape[0]
    rng = np.random.default_rng(seed)
    checked = set(range(B)) if rows is None else set(int(r) for r in rows)
    cells = np.empty((B, 3, 3))
    for b in range(B):
        for _ in range(100):
            A = np.eye(3) + spread * rng.uniform(-1.0, 1.0, (3, 3))
            c = A @ base
            if b not in checked or pc.pbc_margin(R[b : b + 1], c, np.linalg.inv(c))[0] >= 1e-6:
                break
        else:
            raise AssertionError('no cell away from rounding ties for geometry %d' % b)
        cells[b] = c
    return cells


def image_patterns(R, cells):
    """Per geometry, the integer image k = round(L^-1 d) of every pair in its own cell: (B, D, 3)."""
    R = np.asarray(R, dtype=np.float64)
    return np.stack([np.around(pc._pair_frac(R[b : b + 1], np.linalg.inv(cells[b]))[1][0]) for b in range(R.shape[0])])


def assert_cells_wrap_differently(R, cells):
    """Pairs wrap in a good part of the geometries, and into images that differ between geometries."""
    k = image_patterns(R, cells)
    wraps = np.any(k != 0, axis=(1, 2))
    assert np.mean(wraps) >= 0.2, 'too few geometries wrap'
    if R.shape[0] > 1:
        assert len({kb.tobytes() for kb in k}) > 1, 'every geometry wraps into the same images'


def oracle_cells(op, R, cells):
    """(E, F, W) of the oracle Predictor `op` with geometry b in cell cells[b] (cells None: op's own cell)."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * op.n_atoms)
    if cells is None:
        return vc.oracle_virial(op, R)[:3]
    parts = [vc.oracle_virial(vc.with_cell(op, cells[b]), R[b : b + 1])[:3] for b in range(R.shape[0])]
    return tuple(np.concatenate(x) for x in zip(*parts))


class OracleVirialPredictor(object):
    """The oracle with GDMLPredict.predict_virial's interface (NumPy in / out): a stand-in for the engine in the CPU
    tests of the sharded predictors."""

    def __init__(self, model):
        self.op = opredict.Predictor(model)

    def predict_virial(self, R, lattice=None, return_E=True):
        R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * self.op.n_atoms)
        lat = None if lattice is None else np.asarray(lattice, dtype=np.float64)
        if lat is not None and lat.ndim == 3:
            E, F, W = oracle_cells(self.op, R, lat)
        else:
            E, F, W = oracle_cells(self.op if lat is None else vc.with_cell(self.op, lat), R, None)
        return (E, F, W) if return_E else (F, W)


def check_cells(tag, model, op, R, cells, E, F, W, margin=10.0):
    """E, F (check_predict) and W (check_W) of every geometry against the oracle `op` in that geometry's own cell
    (cells None: op's cell), W at `margin` times below tau.  Returns the worst |W err| / scale."""
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3 * op.n_atoms)
    E = None if E is None else np.asarray(E, dtype=np.float64)
    F = np.asarray(F, dtype=np.float64).reshape(R.shape[0], -1)
    W = np.asarray(W, dtype=np.float64).reshape(-1, 3, 3)
    D = model['R_desc'].shape[0]
    k = pc.n_terms(model['R_desc'].shape[1], op.n_perms, D)
    worst = 0.0
    for b in range(R.shape[0]):
        opb = op if cells is None else vc.with_cell(op, cells[b])
        Rb = R[b : b + 1]
        E_ref, F_ref, W_ref, _ = vc.oracle_virial(opb, Rb)
        m = dict(model)
        if opb.lat_and_inv is not None:
            m['lattice'] = opb.lat_and_inv[0]
        else:
            m.pop('lattice', None)
        pc.check_predict(None if E is None else E[b : b + 1], F[b : b + 1], E_ref, F_ref,
                         pc.predict_abs_scale(m, Rb, oracle=opb), k, what='%s row %d' % (tag, b))
        worst = max(worst, vc.check_W(W[b : b + 1], W_ref, vc.virial_abs_scale(m, Rb, opb), k,
                                      what='%s row %d' % (tag, b)))
    print('\n[virial cells bound] %s: %d rows, max|err|/scale %.2e, tau %.2e' % (tag, R.shape[0], worst, pc.tau(k)))
    assert worst <= pc.tau(k) / margin, '%s: less than %gx margin below tau' % (tag, margin)
    return worst
