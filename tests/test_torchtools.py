"""sgdml_b200.torchtools.GDMLTorchPredict: the reference's torch module with autograd through E and F.

forward equals GDMLPredict.predict bit for bit; grad(E.sum(), R) is -F; torch.autograd.gradcheck passes; a force-matching
loss and the dense Hessian (torch.autograd.functional.hessian, and the batched-identity form in one engine call) match
the torch oracle (tests/hvp_oracle.py); third derivatives raise; lat_and_inv decides the cell."""

import os

import numpy as np
import pytest

import hvp_oracle as ho
from conftest import rel_err


@pytest.mark.skipif(os.environ.get('SGDML_B200_EXPECT_GPU') == '1', reason='GPU box')
def test_construction_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip('a GPU is visible')
    from sgdml_b200 import _lib
    from sgdml_b200.torchtools import GDMLTorchPredict

    model, _, _ = ho.fixture_model('n9_m16_s6')
    with pytest.raises(_lib.EngineError, match='no CPU fallback'):
        GDMLTorchPredict(model)


@pytest.fixture(scope='module')
def tt():
    from sgdml_b200 import _lib
    from sgdml_b200 import torchtools

    _lib.require_gpu()
    return torchtools


def _R(Rq, B):
    import torch

    N = Rq.shape[1] // 3
    return torch.from_numpy(np.ascontiguousarray(Rq[:B])).reshape(B, N, 3).cuda()


@pytest.mark.gpu
def test_forward_and_energy_gradient(tt):
    import torch

    import sgdml_b200

    model, Rq, _ = ho.fixture_model('n9_m16_s6')
    mod = tt.GDMLTorchPredict(model)
    R = _R(Rq, 5).requires_grad_()
    E, F = mod(R)
    E0, F0 = sgdml_b200.GDMLPredict(model).predict(Rq[:5])
    assert np.array_equal(E.detach().cpu().numpy(), E0) and np.array_equal(F.detach().cpu().numpy().reshape(5, -1), F0)
    (F_only,) = mod(R, return_E=False)
    assert torch.equal(F_only, F)
    (g,) = torch.autograd.grad(E.sum(), R)
    assert torch.equal(g, -F.detach())
    # other float dtypes are cast to float64
    E32, F32 = mod(R.detach().float())
    assert E32.dtype == torch.float64 and F32.shape == F.shape
    with pytest.raises(ValueError, match='training-index'):
        mod(torch.arange(3, device='cuda'))


@pytest.mark.gpu
def test_gradcheck(tt):
    import torch

    model, Rq, _ = ho.fixture_model('n9_m16_s6')
    mod = tt.GDMLTorchPredict(model)
    R = _R(Rq, 2).requires_grad_()
    assert torch.autograd.gradcheck(mod, (R,))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'ecstr_n6_m8', 'big_n100_m2_s12'])
def test_force_matching_loss_gradient(tt, name):
    import torch

    model, Rq, _ = ho.fixture_model(name)
    mod = tt.GDMLTorchPredict(model)
    B = min(3, Rq.shape[0])
    F0 = torch.from_numpy(np.random.default_rng(0).standard_normal((B, Rq.shape[1]))).cuda()
    R = _R(Rq, B).requires_grad_()
    _, F = mod(R)
    (g,) = torch.autograd.grad(((F.reshape(B, -1) - F0) ** 2).sum(), R)
    to = ho.TorchOracle(model)
    Ro = torch.from_numpy(np.ascontiguousarray(Rq[:B])).requires_grad_()
    (go,) = torch.autograd.grad(((to.ef(Ro)[1] - F0.cpu()) ** 2).sum(), Ro)
    err = rel_err(g.cpu().numpy().reshape(B, -1), go.numpy())
    print('\n[torchtools] %s force-loss gradient against the oracle %.2e' % (name, err))
    assert err <= 1e-8


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['n9_m16_s6', 'big_n100_m2_s12'])
def test_hessian(tt, name):
    import torch

    model, Rq, _ = ho.fixture_model(name)
    mod = tt.GDMLTorchPredict(model)
    N = Rq.shape[1] // 3
    R = _R(Rq, 1)
    H = torch.autograd.functional.hessian(lambda r: mod(r)[0].sum(), R).reshape(3 * N, 3 * N).cpu().numpy()
    # batched identity: one engine call for all 3N rows of -dF/dR
    Rb = R.expand(3 * N, N, 3).clone().requires_grad_()
    _, Fb = mod(Rb)
    eye = torch.eye(3 * N, dtype=torch.float64, device='cuda').reshape(3 * N, N, 3)
    (Hb,) = torch.autograd.grad(Fb, Rb, grad_outputs=-eye)
    Hb = Hb.reshape(3 * N, 3 * N).cpu().numpy()
    H_ref = ho.TorchOracle(model).hessian(Rq[0])
    print('\n[torchtools] %s Hessian: vs batched identity %.2e, vs oracle %.2e, asymmetry %.2e'
          % (name, rel_err(H, Hb), rel_err(H, H_ref), rel_err(H, H.T)))
    assert rel_err(H, Hb) <= 1e-12
    assert rel_err(H, H_ref) <= 1e-8
    assert rel_err(H, H.T) <= 1e-10


@pytest.mark.gpu
def test_third_derivative_raises(tt):
    import torch

    model, Rq, _ = ho.fixture_model('n9_m16_s6')
    mod = tt.GDMLTorchPredict(model)
    R = _R(Rq, 2).requires_grad_()
    _, F = mod(R)
    (g,) = torch.autograd.grad((F * F).sum(), R, create_graph=True)
    with pytest.raises(RuntimeError, match='third derivatives are not supported'):
        torch.autograd.grad(g.sum(), R)


@pytest.mark.gpu
def test_lat_and_inv_decides_the_cell(tt):
    import torch

    import sgdml_b200

    model, Rq, _ = ho.fixture_model('pbc_n6_m8')
    lat = np.asarray(model['lattice'], dtype=np.float64)
    cell = (lat, np.linalg.inv(lat))
    B = Rq.shape[0]
    free = dict(model)
    del free['lattice']
    for mod, ref_model, lai in ((tt.GDMLTorchPredict(model, lat_and_inv=cell), model, cell),
                                (tt.GDMLTorchPredict(model), free, None)):
        R = _R(Rq, B).requires_grad_()
        E, F = mod(R)
        E0, F0 = sgdml_b200.GDMLPredict(ref_model).predict(Rq)
        assert np.array_equal(E.detach().cpu().numpy(), E0)
        assert np.array_equal(F.detach().cpu().numpy().reshape(B, -1), F0)
        V = torch.from_numpy(np.random.default_rng(1).standard_normal((B, Rq.shape[1]))).cuda()
        (g,) = torch.autograd.grad((F.reshape(B, -1) * V).sum(), R)
        ref = ho.TorchOracle(model, lat_and_inv=lai).hvp(Rq, V.cpu().numpy())
        assert rel_err(g.cpu().numpy().reshape(B, -1), ref) <= 1e-8
    # the two cells really differ on these queries
    assert rel_err(sgdml_b200.GDMLPredict(free).predict(Rq)[1], sgdml_b200.GDMLPredict(model).predict(Rq)[1]) > 1e-3
