"""
tools/vxmstub.py -- a test-only `voxelmorph` module for running the reference's labels_to_image_new
(neurite/tf/models.py:920-1301) on tools/tfshim.py.  Used only by tools/gen_golden.py.

voxelmorph is not part of the reference; its layers are provenance 'contract' here, as the st_* fixtures are:
    VecInt / RescaleTransform / ComposeTransform / SpatialTransformer   the oracle's restatements (oracle/interp.py)
    AffineToDenseShift(shape, shift_center=False)                      oracle/affine.py dense_shift (fixed op order);
                                                                        the matrix it receives is kept in LAST_TRANS
    DrawAffineParams                                                    [B, n] draws per kind from the replay queue,
                                                                        none for a zero bound (oracle/affine.py)
    ParamsToAffineMatrix                                                oracle/affine.py affine_matrix
    utils.draw_flip_matrix / draw_swap_matrix                           one U[0, 1) draw [N] each (oracle/affine.py)
"""
import sys
import types

import numpy as np

from oracle import affine as oaff, interp as ointerp
import tfshim
from tfshim import Tensor, A, T

F32 = np.float32
LAST_TRANS = []


class _L:
    def __init__(self, *a, **k):
        self.a, self.k = a, k


class DrawAffineParams(_L):
    """shift, rot, scale, shear: uniform on [-b, b], or normal with SD b (the scale truncated at 2 SD by redrawing
    the whole [B, n] array and keeping the new values where |z| > 2)."""
    def __call__(self, x):
        n, B = self.k['ndims'], A(T(x)).shape[0]
        out = []
        for kind, size in oaff.sizes(n).items():
            b = self.k.get(kind) or 0
            if b == 0:
                out.append(np.zeros((B, size), F32))
                continue
            if not self.k.get('normal_' + kind, False):
                out.append(A(tfshim._uniform((B, size), minval=-b, maxval=b)))
                continue
            z = A(tfshim._normal((B, size)))
            while kind == 'scale' and np.any(np.abs(z) > 2):
                z = np.where(np.abs(z) > 2, A(tfshim._normal((B, size))), z)
            out.append((z * F32(b) + F32(0)).astype(F32))
        return Tensor(np.concatenate(out, 1))


class ParamsToAffineMatrix(_L):
    def __call__(self, p):
        assert self.k.get('deg') and self.k.get('shift_scale') and self.k.get('last_row')
        return Tensor(oaff.affine_matrix(A(T(p)), self.k['ndims']))


class AffineToDenseShift(_L):
    def __call__(self, mat):
        shape = [int(s) for s in self.a[0]]
        assert self.k.get('shift_center') is False
        mat = np.asarray(A(T(mat)), F32)
        LAST_TRANS.append(mat.copy())
        return Tensor(np.stack([oaff.dense_shift(m, shape) for m in mat], 0))


def draw_flip_matrix(grid_shape, shift_center=True, dtype=None, seed=None):
    assert shift_center is False
    u = A(tfshim._uniform((len(grid_shape),)))
    return Tensor(oaff.flip_matrix(u, [int(s) for s in grid_shape]).astype(F32))


def draw_swap_matrix(ndims, dtype=None, seed=None):
    u = A(tfshim._uniform((ndims,)))
    return Tensor(oaff.swap_matrix(u).astype(F32))


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
    utl = types.ModuleType('voxelmorph.utils')
    utl.draw_flip_matrix, utl.draw_swap_matrix = draw_flip_matrix, draw_swap_matrix
    vxm.layers, vxm.utils = lay, utl
    sys.modules['voxelmorph'] = vxm
    sys.modules['voxelmorph.layers'] = lay
    sys.modules['voxelmorph.utils'] = utl
    return vxm


__all__ = ['install', 'tfshim']
