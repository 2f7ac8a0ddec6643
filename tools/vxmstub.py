"""
tools/vxmstub.py -- a test-only `voxelmorph` module for running the reference's labels_to_image_new
(neurite/tf/models.py:920-1301) on tools/tfshim.py.  Used only by tools/gen_golden.py.

voxelmorph is not part of the reference; its layers are provenance 'contract' here, as the st_* fixtures are:
    VecInt / RescaleTransform / ComposeTransform / SpatialTransformer   the oracle's restatements (oracle/interp.py)
    AffineToDenseShift(shape, shift_center=False)                      M[:N] @ [x, 1] - x on the output grid, fp32
    DrawAffineParams                                                    zeros, no draw: the only case in scope
    ParamsToAffineMatrix                                                identity [B, N+1, N+1] for zero parameters
"""
import sys
import types

import numpy as np

from oracle import interp as ointerp
import tfshim
from tfshim import Tensor, A, T

F32 = np.float32


class _L:
    def __init__(self, *a, **k):
        self.a, self.k = a, k


class DrawAffineParams(_L):
    def __call__(self, x):
        n = self.k['ndims']
        return Tensor(np.zeros((A(T(x)).shape[0], 3 * n if n == 2 else 4 * n), F32))


class ParamsToAffineMatrix(_L):
    def __call__(self, p):
        p = A(T(p))
        assert not np.any(p), 'only zero affine parameters are in scope'
        n = self.k['ndims']
        return Tensor(np.broadcast_to(np.eye(n + 1, dtype=F32), (p.shape[0], n + 1, n + 1)).copy())


class AffineToDenseShift(_L):
    def __call__(self, mat):
        shape = [int(s) for s in self.a[0]]
        assert self.k.get('shift_center') is False
        mat = np.asarray(A(T(mat)), F32)
        grid = np.stack(np.meshgrid(*[np.arange(s, dtype=F32) for s in shape], indexing='ij'), -1)
        n = len(shape)
        loc = np.einsum('bij,...j->b...i', mat[:, :n, :n], grid).astype(F32) + mat[:, None, :n, n].reshape(
            (mat.shape[0],) + (1,) * n + (n,))
        return Tensor((loc - grid).astype(F32))


class VecInt(_L):
    def __call__(self, v):
        return Tensor(ointerp.vec_int(np.asarray(A(T(v)), F32), int_steps=self.k['int_steps']))


class RescaleTransform(_L):
    def __call__(self, t):
        return Tensor(ointerp.rescale_transform(np.asarray(A(T(t)), F32), self.k['zoom_factor']))


class ComposeTransform(_L):
    def __call__(self, ts):
        ts = [np.asarray(A(T(t)), F32) for t in ts]
        return Tensor(np.stack([ointerp.compose([t[b] for t in ts]) for b in range(ts[0].shape[0])], 0))


class SpatialTransformer(_L):
    def __call__(self, inputs):
        vol, trf = [np.asarray(A(T(t)), F32) for t in inputs]
        return Tensor(ointerp.spatial_transformer(vol, trf, self.k.get('interp_method', 'linear'),
                                                  fill_value=self.k.get('fill_value')).astype(F32))


def install():
    vxm = types.ModuleType('voxelmorph')
    lay = types.ModuleType('voxelmorph.layers')
    for c in (DrawAffineParams, ParamsToAffineMatrix, AffineToDenseShift, VecInt, RescaleTransform,
              ComposeTransform, SpatialTransformer):
        setattr(lay, c.__name__, c)
    vxm.layers = lay
    sys.modules['voxelmorph'] = vxm
    sys.modules['voxelmorph.layers'] = lay
    return vxm


__all__ = ['install', 'tfshim']
