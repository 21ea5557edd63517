"""The NumPy restatement of the device NPT step (tests/npt_oracle.py) on the CPU: its barostat stream, its reduction
to md_oracle at zero compressibility, and the isothermal-isobaric ensemble it samples -- the ideal gas, a volume-only
energy against a 1-D quadrature, and the virial identity <V (P0 - P_int)> = kT."""

import numpy as np

import md_oracle
import npt_oracle

N_GAS = 6  # atoms
KT = P0 = 1.0


def _cubes(n_rep, vol):
    a = vol ** (1.0 / 3.0)
    return np.tile((a * np.eye(3)).ravel(), (n_rep, 1)), np.tile((np.eye(3) / a).ravel(), (n_rep, 1))


def _volume_forces(B, V1):
    """E(V) = 1/2 B (V - V1)^2 / V1 with F = 0 and W = -V E'(V) I (B = 0: the ideal gas)."""

    def forces(R, cells, cell_invs):
        vol = npt_oracle.det3(cells)
        W = np.zeros((R.shape[0], 9))
        W[:, [0, 4, 8]] = (-vol * B * (vol - V1) / V1)[:, None]
        return 0.5 * B * (vol - V1) ** 2 / V1, np.zeros_like(R), W

    return forces


def _sample(forces, n_rep=200, n_eq=300, n_steps=2000, dt=0.02, tau_p=1.0, seed=1):
    """Volumes and pressures (n_frames, n_rep) every 10 steps after n_eq steps of equilibration (kT = P0 = 1, unit
    masses, friction 1, compressibility 1)."""
    s = np.ones(3 * N_GAS)
    L0, L0inv = _cubes(n_rep, N_GAS + 1.0)
    rng = np.random.default_rng(0)
    R, V = rng.standard_normal((2, n_rep, 3 * N_GAS))
    args = (s, L0, L0inv)
    st, _ = npt_oracle.run(forces, R, V, *args, n_eq, dt, 1.0, KT, P0, 1.0, tau_p, seed=seed)
    _, fr = npt_oracle.run(forces, st['R'], st['V'], *args, n_steps, dt, 1.0, KT, P0, 1.0, tau_p, seed=seed,
                           step0=n_eq, stride=10, eps=st['eps'])
    return npt_oracle.det3(fr['cell']), fr['P']


def _mean_se(x, n_blocks=20):
    """Mean of the (n_frames, n_rep) series and its standard error from batch means over time."""
    b = x.mean(1)[: len(x) // n_blocks * n_blocks].reshape(n_blocks, -1).mean(1)
    return float(b.mean()), float(b.std(ddof=1) / np.sqrt(n_blocks))


def test_barostat_stream_is_apart_and_normal():
    # the O noise's first counter word is a pair index < 2^31, the exchange's 0x80000000 | k with k <= 2^31 - 3
    assert npt_oracle.BARO_WORD > (0x80000000 | (2**31 - 3)) and npt_oracle.BARO_WORD >= 2**31
    eta = npt_oracle.barostat_normal((5 << 32) + 9, np.arange(1000)[:, None], (1 << 32) - 500 + np.arange(1000))
    n = eta.size
    assert abs(eta.mean()) < 5.0 / np.sqrt(n)
    assert abs(eta.var() - 1.0) < 5.0 * np.sqrt(2.0 / n)
    assert abs((eta**4).mean() - 3.0) < 5.0 * np.sqrt(96.0 / n)
    # the barostat normal is the cosine normal of a coordinate pair with the index 0xFFFFFFFF, never drawn by O
    ctr = np.array([npt_oracle.BARO_WORD, 3, 7, 0], dtype=np.uint64)
    u = md_oracle.philox4x32_10(ctr, (11, 0))
    want = np.sqrt(-2.0 * np.log(md_oracle._uniform53(u[0], u[1]))) * np.cos(2.0 * np.pi * md_oracle._uniform53(u[2], u[3]))
    assert npt_oracle.barostat_normal(11, 3, 7) == want


def test_kinetic_order():
    V = np.random.default_rng(3).standard_normal((4, 3 * 137))
    s = np.linspace(0.5, 2.0, V.shape[1])
    assert np.allclose(npt_oracle.kinetic(V, s), md_oracle.kinetic(V, s), rtol=1e-14, atol=0)


def test_zero_compressibility_is_md_run():
    """beta_T = 0: the cells never change and the trajectory is md_oracle.run's bit for bit (E_kin up to its order)."""
    rng = np.random.default_rng(7)
    n_rep, dimi = 3, 3 * 5
    R0, V0 = rng.standard_normal((2, n_rep, dimi))
    s = np.linspace(0.5, 1.5, dimi)
    k = np.linspace(1.0, 3.0, dimi)

    def md_forces(R):
        return 0.5 * (k * R * R).sum(1), -k * R

    def forces(R, cells, cell_invs):
        E, F = md_forces(R)
        return E, F, np.full((R.shape[0], 9), 0.3)  # a virial that would move the cell

    L0, L0inv = _cubes(n_rep, 20.0)
    args = (40, 0.05, 0.7, 0.2)
    ref_final, ref = md_oracle.run(md_forces, R0, V0, s, *args, seed=5, step0=(1 << 32) - 20, stride=10)
    final, fr = npt_oracle.run(forces, R0, V0, s, L0, L0inv, *args, P0=2.0, beta_T=0.0, tau_p=1.0, seed=5,
                               step0=(1 << 32) - 20, stride=10)
    for key in ('R', 'V', 'E_pot'):
        assert np.array_equal(fr[key], ref[key]), key
    assert np.allclose(fr['E_kin'], ref['E_kin'], rtol=1e-14, atol=0)
    assert np.array_equal(final['R'], ref_final[0]) and np.array_equal(final['V'], ref_final[1])
    assert np.all(fr['cell'] == L0) and np.all(final['eps'] == 0.0)


def test_ideal_gas_volume():
    """<V> = (N + 1) kT / P0, within 4 standard errors; N kT / P0 and (N + 2) kT / P0, which a stray +-kT / V in the
    drift would give, lie outside."""
    vol, _ = _sample(_volume_forces(0.0, 1.0))
    m, se = _mean_se(vol)
    print('ideal gas: <V> = %.4f +- %.4f, exact %d' % (m, se, N_GAS + 1))
    assert abs(m - (N_GAS + 1)) < 4.0 * se
    assert abs(m - N_GAS) > 4.0 * se and abs(m - (N_GAS + 2)) > 4.0 * se


def test_volume_energy_against_quadrature():
    """E(V) = 1/2 B (V - V1)^2 / V1: <V> and Var(V) against a quadrature of V^N exp(-beta (P0 V + E(V))), and
    <V (P0 - P_int)> = kT."""
    B, V1 = 2.0, 5.0
    vol, P = _sample(_volume_forces(B, V1), n_steps=4000, dt=0.01, tau_p=2.0)
    x = np.linspace(1e-6, 60.0, 600001)
    w = N_GAS * np.log(x) - (P0 * x + 0.5 * B * (x - V1) ** 2 / V1) / KT
    w = np.exp(w - w.max())
    mean = float((x * w).sum() / w.sum())
    var = float(((x - mean) ** 2 * w).sum() / w.sum())
    m, se = _mean_se(vol)
    v, se_v = _mean_se((vol - mean) ** 2)
    vir, se_vir = _mean_se(vol * (P0 - P))
    print('E(V): <V> = %.4f +- %.4f (%.4f), Var(V) = %.4f +- %.4f (%.4f), <V (P0 - P)> = %.4f +- %.4f'
          % (m, se, mean, v, se_v, var, vir, se_vir))
    assert abs(m - mean) < 4.0 * se
    assert abs(v - var) < 4.0 * se_v
    assert abs(vir - KT) < 4.0 * se_vir
