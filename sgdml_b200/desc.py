"""Host-side mirror of the reference's ``sgdml.utils.desc.Desc`` for the hot path.

Same method names / argument meaning as utils/desc.py:242-539, but every numeric method
runs on the GPU through the C ABI (no NumPy fallback).  ``Desc.perm`` /
``tril_perms_lin`` are the integer host routines of the library (bit-exact).
"""

import numpy as np

from . import _lib


def _as_f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def tril_perms_lin(perms):
    """perms (S, N) int -> tril_perms_lin (S*D,) int64 (train.py:897-904)."""
    perms = np.ascontiguousarray(perms, dtype=np.int64)
    if perms.ndim != 2:
        raise ValueError('perms must be (n_perms, n_atoms)')
    S, N = perms.shape
    out = np.empty(S * (N * (N - 1) // 2), dtype=np.int64)
    _lib.check(_lib.lib().sgdml_b200_tril_perms_lin(_lib.ptr(perms), S, N, _lib.ptr(out)), 'tril_perms_lin')
    return out


class Desc(object):
    def __init__(self, n_atoms, max_processes=None):
        """utils/desc.py:244-286.  `max_processes` is accepted for signature compatibility
        and ignored (descriptors are generated on the GPU)."""
        self.n_atoms = n_atoms
        self.dim_i = 3 * n_atoms
        self.dim = (n_atoms * (n_atoms - 1)) // 2
        self.tril_indices = np.tril_indices(n_atoms, k=-1)
        self.max_processes = max_processes

    def from_R(self, R, lat_and_inv=None, max_processes=None, callback=None):
        """utils/desc.py:288-365: R (M, 3N) -> R_desc (M, D), R_d_desc (M, D, 3).
        A single geometry returns (D,), (D, 3) like the reference (desc.py:329-330)."""
        R = _as_f64(R)
        if R.ndim == 1:
            R = R[None, :]
        R = R.reshape(R.shape[0], -1)
        M = R.shape[0]
        R_desc = np.empty((M, self.dim))
        R_d_desc = np.empty((M, self.dim, 3))
        if lat_and_inv is not None:  # minimum-image convention (desc.py:44-77, 100-108, 200-201)
            lat, lat_inv = (_as_f64(x) for x in lat_and_inv)
            if lat.shape != (3, 3) or lat_inv.shape != (3, 3):
                raise ValueError('lat_and_inv must be a pair of 3 x 3 matrices')
            _lib.check(
                _lib.lib().sgdml_b200_desc_from_R_pbc(
                    _lib.ptr(R), M, self.n_atoms, _lib.ptr(lat), _lib.ptr(lat_inv), _lib.ptr(R_desc), _lib.ptr(R_d_desc),
                    _lib.current_stream(),
                ),
                'desc_from_R_pbc',
            )
        else:
            _lib.check(
                _lib.lib().sgdml_b200_desc_from_R(
                    _lib.ptr(R), M, self.n_atoms, _lib.ptr(R_desc), _lib.ptr(R_d_desc), _lib.current_stream()
                ),
                'desc_from_R',
            )
        if callback is not None:
            callback(M, M)
        if M == 1:
            return R_desc[0], R_d_desc[0]
        return R_desc, R_d_desc

    def d_desc_dot_vec(self, R_d_desc, vecs, overwrite_vecs=False):
        """utils/desc.py:368-385."""
        R_d_desc = _as_f64(R_d_desc)
        vecs = _as_f64(vecs)
        if R_d_desc.ndim == 2:
            R_d_desc = R_d_desc[None]
        if vecs.ndim == 1:
            vecs = vecs[None]
        M = R_d_desc.shape[0]
        vecs = vecs.reshape(M, -1)
        out = np.empty((M, self.dim))
        _lib.check(
            _lib.lib().sgdml_b200_d_desc_dot_vec(
                _lib.ptr(R_d_desc), _lib.ptr(vecs), M, self.n_atoms, _lib.ptr(out), _lib.current_stream()
            ),
            'd_desc_dot_vec',
        )
        return out

    def vec_dot_d_desc(self, R_d_desc, vecs, out=None):
        """utils/desc.py:388-408 (same number of descriptors and vectors, or one of each)."""
        R_d_desc = _as_f64(R_d_desc)
        vecs = _as_f64(vecs)
        if R_d_desc.ndim == 2:
            R_d_desc = R_d_desc[None]
        if vecs.ndim == 1:
            vecs = vecs[None]
        n = max(R_d_desc.shape[0], vecs.shape[0])
        if R_d_desc.shape[0] != n:
            R_d_desc = np.ascontiguousarray(np.broadcast_to(R_d_desc, (n,) + R_d_desc.shape[1:]))
        if vecs.shape[0] != n:
            vecs = np.ascontiguousarray(np.broadcast_to(vecs, (n, vecs.shape[1])))
        res = np.empty((n, self.dim_i))
        _lib.check(
            _lib.lib().sgdml_b200_vec_dot_d_desc(
                _lib.ptr(R_d_desc), _lib.ptr(vecs), n, self.n_atoms, _lib.ptr(res), _lib.current_stream()
            ),
            'vec_dot_d_desc',
        )
        if out is not None:  # desc.py:388-408 fills a caller-provided array in place
            out[...] = res.reshape(out.shape)
            return out
        return res

    @staticmethod
    def perm(perm):
        """utils/desc.py:509-539: atom permutation (N,) -> descriptor permutation (D,)."""
        perm = np.asarray(perm, dtype=np.int64)
        return tril_perms_lin(perm[None, :]).astype(int)
