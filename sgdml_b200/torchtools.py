"""``GDMLTorchPredict`` -- the reference's ``torch.nn.Module`` predictor (sgdml/torchtools.py:395-1128) backed by the
H100 engine, with autograd through energies and forces.

``forward(Rs)`` returns E and F from one engine call.  Both are differentiable with respect to Rs:
``grad(E.sum(), Rs)`` is ``-F``, a loss on the forces backpropagates to the positions through one Hessian-vector
product per geometry (``GDMLPredict.predict_hvp``), and ``torch.autograd.functional.hessian`` works.  There is no
Hessian output: a dense Hessian comes from torch's autograd utilities, or in one engine call as the vector-Jacobian
product of F with the identity rows of a geometry repeated 3N times.  Third derivatives raise ``RuntimeError``.
"""

import numpy as np
import torch

from . import _lib
from .predict import GDMLPredict


class _HVP(torch.autograd.Function):
    """HV = (dF/dR) V per geometry (R, V (B, 3N) float64); the vector-Jacobian product of F, as dF/dR is symmetric."""

    @staticmethod
    def forward(ctx, R, V, pred):
        return pred.predict_hvp(R.contiguous(), V.contiguous())

    @staticmethod
    def backward(ctx, g):
        raise RuntimeError('third derivatives are not supported')


class _EF(torch.autograd.Function):
    """(E (B,), F (B, 3N)) of R (B, 3N) float64 from one `predict` call.  The backward of E is -gE F and that of F is an
    HVP; F enters the backward as a saved OUTPUT of this function, so a gradient taken with create_graph=True is itself
    differentiable through it (Hessians)."""

    @staticmethod
    def forward(ctx, R, pred):
        E, F = pred.predict(R.contiguous())
        ctx.set_materialize_grads(False)  # an unused output costs no HVP
        ctx.pred = pred
        ctx.save_for_backward(R, F)
        return E, F

    @staticmethod
    def backward(ctx, gE, gF):
        R, F = ctx.saved_tensors
        g = None
        if gE is not None:
            g = -gE[:, None] * F
        if gF is not None:
            h = _HVP.apply(R, gF, ctx.pred)
            g = h if g is None else g + h
        return g, None


class GDMLTorchPredict(torch.nn.Module):
    """torchtools.py:395-1128.  Contains no trainable parameters.

    The periodic cell follows the reference: `lat_and_inv` (lattice vectors as columns, and the inverse) decides, and
    `model['lattice']` is ignored; without `lat_and_inv` the model is evaluated as a free molecule.  `batch_size`,
    `n_perm_batches`, `max_memory` and `max_processes` are accepted for signature compatibility; the engine chooses its
    own chunks.  Raises `EngineError` without a GPU, as `GDMLPredict` does."""

    def __init__(
        self,
        model,
        lat_and_inv=None,
        batch_size=None,
        n_perm_batches=1,
        max_memory=None,
        max_processes=None,
        log_level=None,
    ):
        super(GDMLTorchPredict, self).__init__()
        model = dict(model)
        model.pop('lattice', None)
        self._pred = GDMLPredict(model, max_memory=max_memory, max_processes=max_processes, log_level=log_level)
        self.n_atoms = self._pred.n_atoms
        self._lat_and_inv = None
        if lat_and_inv is not None:
            lat = np.ascontiguousarray(lat_and_inv[0], dtype=np.float64)
            lat_inv = np.ascontiguousarray(lat_and_inv[1], dtype=np.float64)
            if lat.shape != (3, 3) or lat_inv.shape != (3, 3):
                raise ValueError('lat_and_inv must hold two 3 x 3 matrices')
            _lib.check(
                _lib.lib().sgdml_b200_model_set_lattice(self._pred._handle, _lib.ptr(lat), _lib.ptr(lat_inv)),
                'model_set_lattice',
            )
            self._lat_and_inv = (lat, lat_inv)

    def forward(self, Rs, return_E=True):
        """Rs (B, N, 3) Cartesian coordinates -> (E (B,), F (B, N, 3)), or (F,) without return_E.  Other float dtypes
        are cast to float64 (a differentiable cast); E and F are float64 on Rs's device."""
        if Rs.dim() == 1:
            raise ValueError(
                'GDMLTorchPredict.forward takes geometries of shape (B, N, 3); the training-index form of the reference '
                'is not supported (use GDMLPredict.predict(R=None))'
            )
        if Rs.dim() != 3 or tuple(Rs.shape[1:]) != (self.n_atoms, 3):
            raise ValueError('Rs must have shape (B, %d, 3)' % self.n_atoms)
        B = Rs.shape[0]
        R = Rs.to(torch.float64).reshape(B, 3 * self.n_atoms)
        E, F = _EF.apply(R, self._pred)
        F = F.reshape(B, self.n_atoms, 3)
        return (E, F) if return_E else (F,)
