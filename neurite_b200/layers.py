"""
neurite_b200.layers -- drop-ins for the hot-path layers of neurite.layers
(adalca/neurite: neurite/tf/layers.py) as torch.nn.Modules on channels-last CUDA tensors.

    Resize / Zoom           layers.py:91-185
    SpatialTransformer      voxelmorph.layers.SpatialTransformer (call sites models.py:806, 1157)
    VecInt, ComposeTransform, RescaleTransform   voxelmorph layers composed from the warp / resize
    LocallyConnected3D      layers.py:811-1197  (implementation 1)
    GaussianBlur, Subsample layers.py:251-443
    RandomCrop              layers.py:446-519
    GaussianNoise, PerlinNoise   layers.py:2305-2508

Constructor arguments, defaults, `get_config()` keys, `compute_output_shape`, weight names
(`kernel`, `bias`) and weight shapes/orderings follow the reference, so configs and
trained weights carry over.  Inputs are [batch, *spatial, channels] like Keras' default.
"""
import math
import os

import numpy as np
import torch

from . import _lib, augment, utils
from ._lib import lib, check, ptr, stream_ptr, i32_array, require_cuda


class _Layer(torch.nn.Module):
    """The slice of the Keras Layer protocol the reference relies on: lazy build on first
    call, get_config round trip, `name`."""

    def __init__(self, name=None, **kwargs):
        super().__init__()
        if kwargs:
            raise TypeError('Keyword argument not understood: %s' % list(kwargs)[0])
        self.name = name or type(self).__name__.lower()
        self.built = False

    def build(self, input_shape):
        self.built = True

    def get_config(self):
        return {'name': self.name}

    @classmethod
    def from_config(cls, config):
        return cls(**config)

    def forward(self, inputs):
        if not self.built:
            shp = [tuple(i.shape) for i in inputs] if isinstance(inputs, (list, tuple)) else tuple(inputs.shape)
            self.build(shp)
        return self.call(inputs)


# ---------------------------------------------------------------------------------------
class Resize(_Layer):
    """N-D Resize (scipy-zoom-like), reference layers.py:91-185."""

    def __init__(self, zoom_factor, interp_method='linear', **kwargs):
        self.zoom_factor = zoom_factor
        self.interp_method = interp_method
        self.ndims = None
        self.inshape = None
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'zoom_factor': self.zoom_factor, 'interp_method': self.interp_method})
        return config

    def build(self, input_shape):
        if isinstance(input_shape[0], (list, tuple)) and len(input_shape) > 1:
            raise Exception('Resize must be called on a list of length 1.')            # :133-134
        if isinstance(input_shape[0], (list, tuple)):
            input_shape = input_shape[0]
        self.ndims = len(input_shape) - 2
        self.inshape = input_shape
        if not isinstance(self.zoom_factor, (list, tuple)):
            self.zoom_factor = [self.zoom_factor] * self.ndims
        else:
            assert len(self.zoom_factor) == self.ndims, \
                'zoom factor length {} does not match number of dimensions {}'.format(
                    len(self.zoom_factor), self.ndims)                                  # :145-147
        self.built = True

    def call(self, inputs):
        if isinstance(inputs, (list, tuple)):
            assert len(inputs) == 1, "inputs has to be len 1. found: %d" % len(inputs)  # :162
            vol = inputs[0]
        else:
            vol = inputs
        vol = vol.reshape((-1,) + tuple(self.inshape[1:]))                              # :168
        if all(z == 1 for z in self.zoom_factor):                                       # utils.py:250-251
            return vol
        # the reference maps utils.resize over the batch serially (:171); one launch here
        return utils._resize_batched(vol, list(self.zoom_factor), self.interp_method)

    def compute_output_shape(self, input_shape):
        output_shape = [input_shape[0]]
        output_shape += [int(input_shape[1:-1][f] * self.zoom_factor[f]) for f in range(self.ndims)]
        output_shape += [input_shape[-1]]
        return tuple(output_shape)


Zoom = Resize


# ---------------------------------------------------------------------------------------
class SpatialTransformer(_Layer):
    """Dense-shift spatial transformer with the voxelmorph call signature
    (SpatialTransformer(interp_method, indexing, single_transform, fill_value, shift_center,
    shape)([vol, trf])).  The reference calls it as vxm.layers.SpatialTransformer at
    neurite/tf/models.py:806-807 and 1157-1159; the arithmetic is
    out[b] = neurite.utils.interpn(vol[b], ndgrid + trf[b]).

    Affine transforms ([B, N, N+1]) are expanded to a dense shift first (thin torch code);
    `halo` is a tiling hint for the shared-memory kernel (expected max |shift| in voxels) and
    never changes results."""

    def __init__(self, interp_method='linear', indexing='ij', single_transform=False,
                 fill_value=None, shift_center=True, shape=None, halo=0, **kwargs):
        self.interp_method = interp_method
        assert indexing in ['ij', 'xy'], "indexing has to be 'ij' (matrix) or 'xy' (cartesian)"
        self.indexing = indexing
        self.single_transform = single_transform
        self.fill_value = fill_value
        self.shift_center = shift_center
        self.shape = shape
        self.halo = halo
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'interp_method': self.interp_method, 'indexing': self.indexing,
                       'single_transform': self.single_transform, 'fill_value': self.fill_value,
                       'shift_center': self.shift_center, 'shape': self.shape})
        return config

    def build(self, input_shape):
        if len(input_shape) != 2 or not isinstance(input_shape[0], (list, tuple)):
            raise Exception('Spatial Transformer must be called on a list of length 2: '
                            'first argument is the image, second is the transform.')
        self.ndims = len(input_shape[0]) - 2
        self.built = True

    def call_host(self, inputs, out=None, chunk=1):
        """[vol, dense shift] as CPU (pinned) tensors -> warped volume on the CPU, with the
        PCIe copies pipelined against the kernel (utils.warp_host)."""
        assert len(inputs) == 2, 'inputs has to be len 2, found: %d' % len(inputs)
        vol, trf = inputs
        if self.indexing == 'xy':
            trf = torch.cat([trf[..., 1:2], trf[..., 0:1], trf[..., 2:]], -1)
        return utils.warp_host(vol, trf, out, self.interp_method, self.fill_value, self.halo, chunk=chunk)

    def _affine_to_dense(self, mat, volshape):
        """[B, N, N+1] affine -> dense shift [B, *volshape, N] (vxm.utils.affine_to_dense_shift)."""
        nd = len(volshape)
        dev = mat.device
        grid = torch.stack(torch.meshgrid(*[torch.arange(s, dtype=torch.float32, device=dev) for s in volshape],
                                          indexing='ij'), -1)                    # [*S, N]
        g = grid
        if self.shift_center:
            g = g - torch.tensor([(s - 1) / 2 for s in volshape], dtype=torch.float32, device=dev)
        flat = torch.cat([g.reshape(-1, nd), torch.ones(g.numel() // nd, 1, device=dev)], 1)   # [V, N+1]
        loc = torch.einsum('bij,vj->bvi', mat[:, :nd, :].to(torch.float32), flat)              # [B, V, N]
        if self.shift_center:
            loc = loc + torch.tensor([(s - 1) / 2 for s in volshape], dtype=torch.float32, device=dev)
        return loc.reshape((mat.shape[0],) + tuple(volshape) + (nd,)) - grid

    def call(self, inputs):
        assert len(inputs) == 2, 'inputs has to be len 2, found: %d' % len(inputs)
        vol, trf = inputs
        nd = vol.dim() - 2
        if trf.dim() == 3 and tuple(trf.shape[1:]) in ((nd, nd + 1), (nd + 1, nd + 1)):
            # affine [B, N, N+1] or the square homogeneous form [B, N+1, N+1] (vxm accepts both; the last row is dropped)
            trf = self._affine_to_dense(trf[:, :nd, :], tuple(vol.shape[1:-1]) if self.shape is None else tuple(self.shape))
        if self.indexing == 'xy':                                              # swap the first two shift channels
            trf = torch.cat([trf[..., 1:2], trf[..., 0:1], trf[..., 2:]], -1)
        if self.single_transform:
            # vxm: the FIRST transform of the batch is applied to every volume, whatever the transform batch size
            trf = trf[:1].expand((vol.shape[0],) + tuple(trf.shape[1:]))
        if tuple(trf.shape[1:-1]) != tuple(vol.shape[1:-1]):
            # output grid differs from the volume grid: go through interpn per batch item (one grid for all of them)
            mesh = utils.volshape_to_ndgrid(trf.shape[1:-1], device=trf.device)
            grid = torch.stack([m.to(torch.float32) for m in mesh], -1)
            return torch.stack([utils.interpn(vol[b], grid + trf[b], self.interp_method, self.fill_value)
                                for b in range(vol.shape[0])], 0)
        return utils._warp_batched(vol, trf, self.interp_method, self.fill_value, halo=self.halo)


# ---------------------------------------------------------------------------------------
# voxelmorph-adjacent transforms that feed the warp (SURVEY.md 8f item 2).  Thin compositions
# of the kernels above; call sites in the reference: neurite/tf/models.py:802-804, 1149.
# ---------------------------------------------------------------------------------------
class VecInt(_Layer):
    """vxm.layers.VecInt: integrate a stationary velocity field by scaling and squaring
    (method 'ss'): v /= 2^int_steps; repeat int_steps times: v += warp(v, v)."""

    def __init__(self, indexing='ij', method='ss', int_steps=7, out_time_pt=1, **kwargs):
        assert indexing in ['ij', 'xy'], "indexing has to be 'ij' (matrix) or 'xy' (cartesian)"
        if method != 'ss':
            raise NotImplementedError("VecInt: only method='ss' (scaling and squaring) is built")
        self.indexing, self.method, self.int_steps, self.out_time_pt = indexing, method, int_steps, out_time_pt
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'indexing': self.indexing, 'method': self.method, 'int_steps': self.int_steps,
                       'out_time_pt': self.out_time_pt})
        return config

    def call(self, inputs):
        v = inputs[0] if isinstance(inputs, (list, tuple)) else inputs
        if self.indexing == 'xy':
            v = torch.cat([v[..., 1:2], v[..., 0:1], v[..., 2:]], -1)
        v = v * self.out_time_pt if self.out_time_pt != 1 else v
        v = v / (2 ** self.int_steps)
        for _ in range(self.int_steps):
            v = v + utils._warp_batched(v, v, 'linear', None)
        return v


class ComposeTransform(_Layer):
    """vxm.layers.ComposeTransform for dense shifts: T = t_0 o t_1 o ... (the right-most
    transform is applied first): curr = t_last; curr = curr + warp(t_next, curr)."""

    def __init__(self, interp_method='linear', shift_center=True, indexing='ij', **kwargs):
        self.interp_method, self.shift_center, self.indexing = interp_method, shift_center, indexing
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'interp_method': self.interp_method, 'shift_center': self.shift_center,
                       'indexing': self.indexing})
        return config

    def call(self, transforms):
        if not isinstance(transforms, (list, tuple)) or len(transforms) < 2:
            raise ValueError('ComposeTransform must be called on a list of at least two transforms')
        for t in transforms:
            if t.dim() == 3:
                raise NotImplementedError('ComposeTransform: affine inputs are not built; expand them with '
                                          'SpatialTransformer._affine_to_dense first')
        curr = transforms[-1]
        for nxt in reversed(transforms[:-1]):
            curr = curr + utils._warp_batched(nxt, curr, self.interp_method, None)
        return curr


class RescaleTransform(_Layer):
    """vxm.layers.RescaleTransform for dense shifts: resize the field by zoom_factor and scale
    its values by the same factor (values first when up-sampling, resize first when down-sampling)."""

    def __init__(self, zoom_factor, interp_method='linear', **kwargs):
        self.zoom_factor, self.interp_method = zoom_factor, interp_method
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'zoom_factor': self.zoom_factor, 'interp_method': self.interp_method})
        return config

    def call(self, trf):
        ndims = trf.dim() - 2
        if self.zoom_factor < 1:
            return utils._resize_batched(trf, [self.zoom_factor] * ndims, self.interp_method) * self.zoom_factor
        return utils._resize_batched(trf * self.zoom_factor, [self.zoom_factor] * ndims, self.interp_method)


# ---------------------------------------------------------------------------------------
def _normalize_tuple(value, n, name):
    if isinstance(value, int):
        return (value,) * n
    value = tuple(value)
    if len(value) != n:
        raise ValueError('The `%s` argument must be a tuple of %d integers. Received: %s' % (name, n, value))
    return tuple(int(v) for v in value)


def conv_output_length(input_length, filter_size, padding, stride):
    """keras conv_utils.conv_output_length for 'valid'/'same' (layers.py:963-968)."""
    if input_length is None:
        return None
    out = input_length if padding == 'same' else input_length - filter_size + 1
    return (out + stride - 1) // stride


class LocallyConnected3D(_Layer):
    """Unshared-weight 3-D convolution, reference layers.py:811-1197, implementation 1.

    kernel: [P, k0*k1*k2*Cin, filters] with P = o0*o1*o2 row-major (layers.py:974-984);
    bias:   [o0, o1, o2, filters] (layers.py:1034-1040)."""

    def __init__(self, filters, kernel_size, strides=(1, 1, 1), padding='valid', data_format=None,
                 activation=None, use_bias=True, kernel_initializer='glorot_uniform',
                 bias_initializer='zeros', kernel_regularizer=None, bias_regularizer=None,
                 activity_regularizer=None, kernel_constraint=None, bias_constraint=None,
                 implementation=1, **kwargs):
        super().__init__(**kwargs)
        self.filters = filters
        self.kernel_size = _normalize_tuple(kernel_size, 3, 'kernel_size')
        self.strides = _normalize_tuple(strides, 3, 'strides')
        self.padding = padding.lower()
        if self.padding != 'valid' and implementation == 1:
            raise ValueError('Invalid border mode for LocallyConnected3D '
                             '(only "valid" is supported if implementation is 1): ' + padding)   # :934-936
        self.data_format = 'channels_last' if data_format is None else data_format.lower()
        if self.data_format not in ('channels_last', 'channels_first'):
            raise ValueError('Unknown data_format: ' + str(data_format))
        if activation is not None and not callable(activation) and activation not in _lib.ACTIVATIONS:
            raise ValueError('Unknown activation function: %s' % activation)
        self.activation = activation
        self.use_bias = use_bias
        self.kernel_initializer = kernel_initializer
        self.bias_initializer = bias_initializer
        self.kernel_regularizer = kernel_regularizer
        self.bias_regularizer = bias_regularizer
        self.activity_regularizer = activity_regularizer
        self.kernel_constraint = kernel_constraint
        self.bias_constraint = bias_constraint
        if implementation not in (1, 2, 3):
            raise ValueError('Unrecognized implementation mode: %d.' % implementation)            # :1030-1032
        if implementation != 1 and self.padding != 'valid':
            # implementations 2 / 3 also allow 'same' in the reference (masks / index lists over the padded
            # geometry, layers.py:986-1028); here they are weight-LAYOUT variants feeding the implementation-1
            # kernel, which is 'valid' only
            raise NotImplementedError("LocallyConnected3D implementations 2 / 3 are built for padding='valid'")
        self.implementation = implementation
        self.kernel = None
        self.bias = None

    def build(self, input_shape):
        input_shape = tuple(input_shape)
        if len(input_shape) != 5:
            raise ValueError('LocallyConnected3D expects a 5D input, got shape ' + str(input_shape))
        if self.data_format == 'channels_last':
            input_row, input_col, input_z = input_shape[1:-1]
            input_filter = input_shape[4]
        else:
            input_row, input_col, input_z = input_shape[2:]
            input_filter = input_shape[1]
        if input_row is None or input_col is None or input_z is None:
            raise ValueError('The spatial dimensions of the inputs to  a LocallyConnected3D layer '
                             'should be fully-defined, but layer received the inputs shape ' + str(input_shape))
        self.output_row = conv_output_length(input_row, self.kernel_size[0], self.padding, self.strides[0])
        self.output_col = conv_output_length(input_col, self.kernel_size[1], self.padding, self.strides[1])
        self.output_z = conv_output_length(input_z, self.kernel_size[2], self.padding, self.strides[2])
        self.input_filter = input_filter
        self.input_spatial = (input_row, input_col, input_z)
        P = self.output_row * self.output_col * self.output_z
        F = self.kernel_size[0] * self.kernel_size[1] * self.kernel_size[2] * input_filter
        self.impl1_kernel_shape = (P, F, self.filters)
        if self.implementation == 1:
            self.kernel_shape = self.impl1_kernel_shape                                          # :974-977
        elif self.implementation == 2:
            # dense input x output weight, masked to the local connectivity (:986-1006)
            if self.data_format == 'channels_first':
                self.kernel_shape = (input_filter, input_row, input_col, input_z,
                                     self.filters, self.output_row, self.output_col, self.output_z)
            else:
                self.kernel_shape = (input_row, input_col, input_z, input_filter,
                                     self.output_row, self.output_col, self.output_z, self.filters)
            if int(np.prod(self.kernel_shape)) > 2 ** 31:
                raise ValueError('implementation 2 stores a dense %s weight: too large' % (self.kernel_shape,))
        else:
            # one weight per connected (output, input) pair, ordered by the sorted index pairs (:1008-1028)
            self.kernel_shape = (P * F * self.filters,)
        if self.kernel is None:
            kernel = torch.empty(self.kernel_shape, dtype=torch.float32)
            if self.implementation == 1:
                self._init(kernel, self.kernel_initializer, fan_in=F, fan_out=self.filters)
            else:
                k1 = torch.empty(self.impl1_kernel_shape, dtype=torch.float32)
                self._init(k1, self.kernel_initializer, fan_in=F, fan_out=self.filters)
                kernel = lc3d_kernel_to_impl(k1, self.implementation, self.input_spatial, input_filter, self.kernel_size,
                                             self.strides, self.data_format)
            self.kernel = torch.nn.Parameter(kernel)
        if self.use_bias and self.bias is None:
            bias = torch.empty((self.output_row, self.output_col, self.output_z, self.filters), dtype=torch.float32)
            self._init(bias, self.bias_initializer, fan_in=1, fan_out=1)
            self.bias = torch.nn.Parameter(bias)
        self.built = True

    @staticmethod
    def _init(t, initializer, fan_in, fan_out):
        if callable(initializer):
            initializer(t)
        elif initializer == 'zeros':
            t.zero_()
        elif initializer == 'ones':
            t.fill_(1.)
        elif initializer == 'glorot_uniform':
            # keras VarianceScaling(scale=1, mode='fan_avg', 'uniform') with keras' fan
            # computation for rank-3 shapes: receptive field = shape[0]
            rf = t.shape[0] if t.dim() == 3 else 1
            limit = math.sqrt(6.0 / (rf * fan_in + rf * fan_out)) if t.dim() == 3 else math.sqrt(6.0 / (fan_in + fan_out))
            t.uniform_(-limit, limit)
        else:
            raise ValueError('Unknown initializer: %s' % initializer)

    def compute_output_shape(self, input_shape):
        if self.data_format == 'channels_first':
            rows, cols, z = input_shape[2], input_shape[3], input_shape[4]
        else:
            rows, cols, z = input_shape[1], input_shape[2], input_shape[3]
        rows = conv_output_length(rows, self.kernel_size[0], self.padding, self.strides[0])
        cols = conv_output_length(cols, self.kernel_size[1], self.padding, self.strides[1])
        z = conv_output_length(z, self.kernel_size[2], self.padding, self.strides[2])
        if self.data_format == 'channels_first':
            return (input_shape[0], self.filters, rows, cols, z)
        return (input_shape[0], rows, cols, z, self.filters)

    def call(self, inputs):
        kernel = self.kernel
        if self.implementation != 1:
            # implementations 2 / 3 (layers.py:1080-1091): the same unshared map stored as a masked dense matrix /
            # as the values of a sparse matrix.  Re-indexed (torch gather: differentiable, so the parameter keeps
            # the reference's shape and ordering and trained weights load as they are) into the [P, F, Cout] blocks
            # the streaming kernel consumes.
            kernel = lc3d_kernel_from_impl(kernel, self.implementation, self.input_spatial, self.input_filter,
                                           self.filters, self.kernel_size, self.strides, self.data_format)
        return local_conv3d(inputs, kernel, self.bias if self.use_bias else None, self.kernel_size,
                            self.strides, (self.output_row, self.output_col, self.output_z),
                            self.data_format, self.activation)

    def get_config(self):
        config = {
            'filters': self.filters, 'kernel_size': self.kernel_size, 'strides': self.strides,
            'padding': self.padding, 'data_format': self.data_format, 'activation': self.activation,
            'use_bias': self.use_bias, 'kernel_initializer': self.kernel_initializer,
            'bias_initializer': self.bias_initializer, 'kernel_regularizer': self.kernel_regularizer,
            'bias_regularizer': self.bias_regularizer, 'activity_regularizer': self.activity_regularizer,
            'kernel_constraint': self.kernel_constraint, 'bias_constraint': self.bias_constraint,
            'implementation': self.implementation,
        }
        base_config = super().get_config()
        return dict(list(base_config.items()) + list(config.items()))


_TORCH_ACT = {None: None, 'linear': None, 'relu': torch.relu, 'sigmoid': torch.sigmoid, 'tanh': torch.tanh}


def _lc3d_impl2_index(input_spatial, Cin, Cout, kernel_size, strides, data_format, device):
    """Flat indices into the implementation-2 weight (dense input x output, layers.py:986-992) of the entries that
    form the implementation-1 kernel [P, F, Cout] ('valid' padding: patch voxel = position * stride + tap)."""
    I, K, St = list(input_spatial), list(kernel_size), list(strides)
    O = [(I[d] - K[d]) // St[d] + 1 for d in range(3)]
    ar = lambda n: torch.arange(n, device=device)      # noqa: E731
    p = torch.stack(torch.meshgrid(ar(O[0]), ar(O[1]), ar(O[2]), indexing='ij'), -1).reshape(-1, 1, 1, 3)      # [P,1,1,3]
    if data_format == 'channels_first':               # feature j = ((c*k0+i0)*k1+i1)*k2+i2
        c, i0, i1, i2 = torch.meshgrid(ar(Cin), ar(K[0]), ar(K[1]), ar(K[2]), indexing='ij')
    else:                                             # feature j = ((i0*k1+i1)*k2+i2)*Cin + c
        i0, i1, i2, c = torch.meshgrid(ar(K[0]), ar(K[1]), ar(K[2]), ar(Cin), indexing='ij')
    tap = torch.stack([i0, i1, i2], -1).reshape(1, -1, 1, 3)
    c = c.reshape(1, -1, 1)
    f = ar(Cout).reshape(1, 1, -1)
    q = p * torch.tensor(St, device=device) + tap                                                            # [P,F,1,3]
    if data_format == 'channels_first':
        dims = (Cin, I[0], I[1], I[2], Cout, O[0], O[1], O[2])
        sub = (c, q[..., 0], q[..., 1], q[..., 2], f, p[..., 0], p[..., 1], p[..., 2])
    else:
        dims = (I[0], I[1], I[2], Cin, O[0], O[1], O[2], Cout)
        sub = (q[..., 0], q[..., 1], q[..., 2], c, p[..., 0], p[..., 1], p[..., 2], f)
    flat = torch.zeros((), dtype=torch.int64, device=device)
    for s, n in zip(sub, dims):
        flat = flat * n + s
    return flat                                                                                              # [P,F,Cout]


def lc3d_kernel_from_impl(kernel, implementation, input_spatial, Cin, Cout, kernel_size, strides,
                          data_format='channels_last'):
    """Weights stored the way LocallyConnected3D implementation 2 or 3 stores them (reference layers.py:986-1028)
    -> the implementation-1 kernel [P, k0*k1*k2*Cin, Cout] (layers.py:974-984).  padding 'valid'.

    impl 2: dense (input..., output...) tensor, channels placed like the data; only the connected entries are used
            (the reference multiplies by a 0/1 mask, :1260-1304).
    impl 3: 1-D vector of the connected entries in the order of sorted (out_flat, in_flat) index pairs
            (conv_kernel_idxs :1346-1434): for channels_last out_flat = ravel(p, f), in_flat = ravel(q, c), which is
            [P, Cout, F] row-major with F in implementation-1 feature order; channels_first: [Cout, P, F]."""
    K, St = list(kernel_size), list(strides)
    O = [(int(input_spatial[d]) - K[d]) // St[d] + 1 for d in range(3)]
    P, F = O[0] * O[1] * O[2], K[0] * K[1] * K[2] * Cin
    if implementation == 1:
        return kernel
    if implementation == 3:
        if kernel.numel() != P * F * Cout:
            raise ValueError('implementation-3 kernel has %d weights, expected %d' % (kernel.numel(), P * F * Cout))
        if data_format == 'channels_first':
            return kernel.reshape(Cout, P, F).permute(1, 2, 0).contiguous()
        return kernel.reshape(P, Cout, F).permute(0, 2, 1).contiguous()
    if implementation == 2:
        idx = _lc3d_impl2_index(input_spatial, Cin, Cout, K, St, data_format, kernel.device)
        return kernel.reshape(-1)[idx]
    raise ValueError('Unrecognized implementation mode: %d.' % implementation)


def lc3d_kernel_to_impl(kernel1, implementation, input_spatial, Cin, kernel_size, strides, data_format='channels_last'):
    """Inverse of lc3d_kernel_from_impl: an implementation-1 kernel [P, F, Cout] in the layout of implementation 2
    (dense, zeros at unconnected entries) or 3 (sorted sparse values)."""
    K, St = list(kernel_size), list(strides)
    O = [(int(input_spatial[d]) - K[d]) // St[d] + 1 for d in range(3)]
    P, F, Cout = kernel1.shape
    if implementation == 1:
        return kernel1
    if implementation == 3:
        if data_format == 'channels_first':
            return kernel1.permute(2, 0, 1).reshape(-1).contiguous()
        return kernel1.permute(0, 2, 1).reshape(-1).contiguous()
    I = [int(s) for s in input_spatial]
    shape = (Cin, I[0], I[1], I[2], Cout, O[0], O[1], O[2]) if data_format == 'channels_first' \
        else (I[0], I[1], I[2], Cin, O[0], O[1], O[2], Cout)
    dense = torch.zeros(int(np.prod(shape)), dtype=kernel1.dtype, device=kernel1.device)
    dense[_lc3d_impl2_index(input_spatial, Cin, Cout, K, St, data_format, kernel1.device).reshape(-1)] = kernel1.reshape(-1)
    return dense.reshape(shape)


def _lc3d_raw(x, k, b, kernel_size, strides, feature_order, act_id, p0, p_count):
    B, Cin, Cout = x.shape[0], x.shape[-1], k.shape[-1]
    out = torch.empty((B, p_count, Cout), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.nrt_lc3d_fwd_f32(ptr(x), ptr(k), ptr(b), ptr(out), B, i32_array(x.shape[1:4]), Cin, Cout,
                                   i32_array(kernel_size), i32_array(strides), feature_order, act_id,
                                   int(p0), int(p_count), stream_ptr(x.device)))
    return out


class _LocalConv3dFn(torch.autograd.Function):
    """autograd shell around nrt_lc3d_fwd_f32 / nrt_lc3d_bwd_f32 (linear activation inside;
    the activation, if any, is applied by torch on the result so its derivative is torch's)."""

    @staticmethod
    def forward(ctx, x, k, b, kernel_size, strides, feature_order, p0, p_count):
        ctx.save_for_backward(x, k)
        ctx.args = (tuple(kernel_size), tuple(strides), feature_order, p0, p_count, b is not None)
        return _lc3d_raw(x.detach(), k.detach(), None if b is None else b.detach(), kernel_size, strides,
                         feature_order, 0, p0, p_count)

    @staticmethod
    def backward(ctx, g):
        x, k = ctx.saved_tensors
        kernel_size, strides, feature_order, p0, p_count, has_bias = ctx.args
        g = g.contiguous().to(torch.float32)
        gx = torch.zeros_like(x) if ctx.needs_input_grad[0] else None
        gk = torch.empty_like(k) if ctx.needs_input_grad[1] else None
        if gx is not None or gk is not None:
            with torch.cuda.device(x.device):
                check(lib.nrt_lc3d_bwd_f32(ptr(x), ptr(k), ptr(g), ptr(gx), ptr(gk), x.shape[0], i32_array(x.shape[1:4]),
                                           x.shape[-1], k.shape[-1], i32_array(kernel_size), i32_array(strides),
                                           feature_order, int(p0), int(p_count), stream_ptr(x.device)))
        gb = g.sum(0) if (has_bias and ctx.needs_input_grad[2]) else None
        return gx, gk, gb, None, None, None, None, None


def local_conv3d(inputs, kernel, bias, kernel_size, strides, output_shape, data_format='channels_last',
                 activation=None, p0=0, p_count=None):
    """LocallyConnected3D.local_conv + bias + activation (layers.py:1126-1197, 1098-1101).

    inputs [B,I0,I1,I2,Cin] (channels_last) or [B,Cin,I0,I1,I2] (channels_first);
    kernel [P,F,Cout]; bias [o0,o1,o2,Cout] or None.  p0/p_count select a contiguous range
    of output positions (position sharding; kernel/bias then hold only that range)."""
    if data_format not in {'channels_first', 'channels_last'}:
        raise ValueError('Unknown data_format: ' + str(data_format))
    require_cuda(inputs, kernel, bias)
    x = inputs.to(torch.float32)
    if data_format == 'channels_first':
        x = x.permute(0, 2, 3, 4, 1)
    x = x.contiguous()
    k = kernel.to(torch.float32).contiguous()
    B, Cout = x.shape[0], k.shape[-1]
    P = int(np.prod(output_shape))
    if p_count is None:
        p_count = P - p0
    b = None if bias is None else bias.to(torch.float32).contiguous().reshape(-1, Cout)
    if b is not None and data_format == 'channels_first':
        # K.bias_add(..., 'channels_first') adds reshape(bias, (1, C, o0, o1, o2)): a RAW reshape of the
        # [o0,o1,o2,C] weight (layers.py:1098-1099 + keras/backend.py), so output[b, f, p] gets bias.flat[f*P + p]
        if p_count != P:
            raise NotImplementedError('channels_first bias under position sharding: the raw-reshape rule needs the whole bias')
        b = b.reshape(Cout, P).t().contiguous()
    feature_order = 1 if data_format == 'channels_first' else 0
    needs_grad = torch.is_grad_enabled() and (x.requires_grad or k.requires_grad or (b is not None and b.requires_grad))
    if needs_grad:
        out = _LocalConv3dFn.apply(x, k, b, tuple(kernel_size), tuple(strides), feature_order, int(p0), int(p_count))
        post = activation if callable(activation) else _TORCH_ACT[activation]
    else:
        fused = activation if (activation is None or isinstance(activation, str)) else None
        out = _lc3d_raw(x, k.detach(), None if b is None else b.detach(), kernel_size, strides, feature_order,
                        _lib.ACTIVATIONS[fused], p0, p_count)
        post = activation if callable(activation) else None
    if p_count == P:
        out = out.reshape((B,) + tuple(output_shape) + (Cout,))
        if data_format == 'channels_first':
            out = out.permute(0, 4, 1, 2, 3).contiguous()
    if post is not None:
        out = post(out)
    return out


# ---------------------------------------------------------------------------------------
class GaussianBlur(_Layer):
    """Blur a tensor [B, *space, C] with a separable Gaussian, reference layers.py:251-364.
    Isotropic or anisotropic, optionally with SDs drawn per call (`random=True`)."""

    def __init__(self, sigma=None, level=None, random=False, min_sigma=0, isotropic=False, seed=None, **kwargs):
        import warnings
        assert sigma is not None or level is not None, 'sigma or level must be provided'
        assert not (sigma is not None and level is not None), 'only sigma or level must be provided'
        if level is not None:
            warnings.warn('The `level` argument to ne.layers.GaussianBlur is deprecated and will '
                          'be removed in a future version. Please use `sigma` instead.')
            if level < 1:
                raise ValueError('Gaussian blur level must not be less than 1')
            if random:
                raise ValueError('level argument incompatible with random blurring')
        if isotropic and not random:
            raise ValueError('For non-random blurring, isotropy is implicitly controlled by the '
                             'number of sigmas provided. Set `isotropic` only for random blur.')
        # (the reference overwrites the level-derived sigma with `sigma` -- None -- at :305; a layer
        #  built from `level` then fails in build().  Here `level` keeps its documented meaning.)
        self.sigma = sigma if sigma is not None else (level - 1) ** 2
        self.random = random
        self.min_sigma = min_sigma
        self.isotropic = isotropic
        self.seed = seed
        self._calls = 0
        self._kernel_cache = {}
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'sigma': self.sigma, 'random': self.random, 'min_sigma': self.min_sigma,
                       'isotropic': self.isotropic, 'seed': self.seed})
        return config

    def _normalize_sigma(self, sigma, ndims):
        sigma = np.ravel(sigma).tolist()
        if len(sigma) not in (1, ndims):
            raise ValueError(f'1 or {ndims} sigmas expected in {ndims}D space, got {len(sigma)}')
        if any(s < 0 for s in sigma):
            raise ValueError('Gaussian blur sigma must not be less than 0')
        if len(sigma) > 1 and self.isotropic:
            raise ValueError(f'random isotropic blur requires a single sigma, got {len(sigma)}')
        if len(sigma) == 1:
            sigma = sigma * ndims
        return sigma

    def build(self, input_shape):
        ndims = len(input_shape) - 2
        self.sigma = self._normalize_sigma(self.sigma, ndims)
        self.min_sigma = self._normalize_sigma(self.min_sigma, ndims)
        if self.isotropic and self.random:
            self.sigma = self.sigma[:1]
            self.min_sigma = self.min_sigma[:1]
        super().build(input_shape)

    def call(self, x):
        if not any(s > 0 for s in self.sigma):
            return x
        if not self.random:
            # fixed SDs: the 1-D kernels are built once per device and stay resident
            key = (x.device.type, x.device.index)
            kernel = self._kernel_cache.get(key)
            if kernel is None:
                kernel = utils.gaussian_kernel(sigma=self.sigma, separate=True, device=x.device)
                kernel = kernel if isinstance(kernel, list) else [kernel]
                self._kernel_cache[key] = kernel
            # an axis with sigma 0 gets the 1-tap kernel [1.0] (utils.py:628-633): x * 1 == x, skip the pass
            axes = [i for i, sg in enumerate(self.sigma) if sg > 0]
            return utils.separable_conv(x, [kernel[i] for i in axes], axis=axes, batched=True)
        seed = None if self.seed is None else self.seed + self._calls       # a fresh draw per call
        self._calls += 1
        kernel = utils.gaussian_kernel(sigma=self.sigma, random=True, min_sigma=self.min_sigma,
                                       separate=True, seed=seed)
        kernel = kernel if isinstance(kernel, list) else [kernel]
        return utils.separable_conv(x, kernel, batched=True)

    def compute_output_shape(self, input_shape):
        return tuple(input_shape)


class Subsample(_Layer):
    """Subsample along one randomly drawn spatial axis with nearest neighbours and optionally
    upsample again, reference layers.py:367-443."""

    def __init__(self, stride_min=1, stride_max=8, axes=None, prob=1, upsample=True, seed=None, **kwargs):
        self.stride_min = stride_min
        self.stride_max = stride_max
        self.axes = axes
        self.prob = prob
        self.upsample = upsample
        self.seed = seed
        self._calls = 0
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'stride_min': self.stride_min, 'stride_max': self.stride_max, 'axes': self.axes,
                       'prob': self.prob, 'upsample': self.upsample, 'seed': self.seed})
        return config

    def build(self, input_shape):
        ndims = len(input_shape) - 2
        assert ndims in (1, 2, 3), 'only 1D, 2D, or 3D supported'
        allowed = list(range(1, ndims + 1))
        if self.axes is None:
            axes = allowed
        else:
            axes = [int(a) % len(input_shape) for a in np.ravel(self.axes)]
            if any(a not in allowed for a in axes):
                raise ValueError(f'axes {self.axes} not in allowed spatial axes {allowed}')
        self.axes = axes
        super().build(input_shape)

    def call(self, x):
        if self.prob == 0 or self.stride_max == 1:
            return x
        seed = None if self.seed is None else self.seed + self._calls
        self._calls += 1
        return utils.subsample_axis(x, stride_min=self.stride_min, stride_max=self.stride_max, axes=self.axes,
                                    prob=self.prob, upsample=self.upsample, seed=seed)


def _crop_window(x, axis, lo, hi):
    """x * mask with mask 1 on [lo, hi) along `axis` (nrt_crop_window_{f32,i32}); fp32 or int32 x."""
    shp = list(x.shape)
    outer = int(np.prod(shp[:axis], dtype=np.int64))
    inner = int(np.prod(shp[axis + 1:], dtype=np.int64))
    out = torch.empty_like(x, memory_format=torch.contiguous_format)
    fn = lib.nrt_crop_window_f32 if x.dtype == torch.float32 else lib.nrt_crop_window_i32
    with torch.cuda.device(x.device):
        check(fn(ptr(x), outer, shp[axis], inner, int(lo), int(hi), ptr(out), stream_ptr(x.device)))
    return out


class _CropFn(torch.autograd.Function):
    """x * mask; the gradient is the upstream gradient times the same mask."""

    @staticmethod
    def forward(ctx, x, axis, lo, hi):
        ctx.window = (axis, lo, hi)
        return _crop_window(x.contiguous(), axis, lo, hi)

    @staticmethod
    def backward(ctx, g):
        return _crop_window(g.to(torch.float32).contiguous(), *ctx.window), None, None, None


class RandomCrop(_Layer):
    """Crop the content of a tensor [B, *space, C] by multiplying with a binary mask that is 1 on a random index
    range of one random spatial axis, reference layers.py:446-519 with augment.draw_crop_mask.  fp32 or int32
    input.  Randomness: see neurite_b200/augment.py; a layer with a seed draws with `seed + number of earlier
    calls`.  The mask is applied by nrt_crop_window_{f32,i32}; the gradient is the same mask."""

    def __init__(self, crop_min=0, crop_max=0.5, axis=None, prob=1, bilateral=False, seed=None, **kwargs):
        self.crop_min = crop_min
        self.crop_max = crop_max
        self.axis = axis
        self.prob = prob
        self.bilateral = bilateral
        self.seed = seed
        self._calls = 0
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'crop_min': self.crop_min, 'crop_max': self.crop_max, 'axis': self.axis, 'prob': self.prob,
                       'bilateral': self.bilateral, 'seed': self.seed})
        return config

    def build(self, input_shape):
        ndims = len(input_shape) - 2
        self.axis = augment.normalize_axes(self.axis, input_shape, range(1, ndims + 1), none_means_all=True)
        super().build(input_shape)

    def _draw(self, shape):
        """(axis, lo, hi) of the next call."""
        seed = None if self.seed is None else self.seed + self._calls
        self._calls += 1
        return augment._draw_crop(list(shape), self.crop_min, self.crop_max, self.axis, self.prob, self.bilateral,
                                  seed)

    def call(self, x):
        if self.prob == 0:
            return x
        require_cuda(x)
        if x.dtype not in (torch.float32, torch.int32):
            raise NotImplementedError(f'RandomCrop: fp32 or int32 input, got {x.dtype}')
        axis, lo, hi = self._draw(x.shape)
        if x.dtype == torch.int32:
            return _crop_window(x.contiguous(), axis, lo, hi)
        return _CropFn.apply(x, axis, lo, hi)


# ---------------------------------------------------------------------------------------
class _NoiseAddFn(torch.autograd.Function):
    """x + noise in one pass (nrt_philox_normal_f32 reads x and writes the output); the noise does not depend
    on x, so the gradient is the identity."""

    @staticmethod
    def forward(ctx, x32, key, shape_sd, table, scale):
        out = torch.empty_like(x32)
        with torch.cuda.device(x32.device):
            check(lib.nrt_philox_normal_f32(key, i32_array(x32.shape), i32_array(shape_sd), x32.dim(), ptr(table),
                                            ptr(scale), ptr(x32), ptr(out), stream_ptr(x32.device)))
        return out

    @staticmethod
    def backward(ctx, g):
        return g, None, None, None, None


class GaussianNoise(_Layer):
    """Draw an SD from U[noise_min, noise_max] per index along `axes` and add N(0, SD) noise to the input, or
    return the noise alone, reference layers.py:2305-2403.  With `absolute=False` the SD is relative to
    max |x| over the whole tensor (computed on the device).  Randomness: see neurite_b200/augment.py; a layer
    with a seed draws with `seed + number of earlier calls`."""

    def __init__(self, noise_min=0.01, noise_max=0.10, noise_only=False, absolute=False, axes=(0, -1), seed=None,
                 **kwargs):
        self.noise_min = noise_min
        self.noise_max = noise_max
        self.noise_only = noise_only
        self.absolute = absolute
        self.axes = axes
        self.seed = seed
        self._calls = 0
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'noise_min': self.noise_min, 'noise_max': self.noise_max, 'noise_only': self.noise_only,
                       'absolute': self.absolute, 'axes': self.axes, 'seed': self.seed})
        return config

    def build(self, input_shape):
        num_dim = len(input_shape)
        self.axes = np.ravel(self.axes)
        self.axes = [int(ax) + num_dim if ax < 0 else int(ax) for ax in self.axes]
        assert all(0 <= ax < num_dim for ax in self.axes), 'invalid axes'
        super().build(input_shape)

    def call(self, x):
        if self.noise_max == 0 and not self.noise_only:
            return x
        if x.is_complex():
            raise NotImplementedError('GaussianNoise: complex inputs are not supported')
        assert x.dtype.is_floating_point, 'non-FP output type'
        require_cuda(x)
        if x.requires_grad and not self.absolute and torch.is_grad_enabled():
            raise RuntimeError('GaussianNoise(absolute=False) has no gradient path through max|x|; '
                               'pass a detached input or use absolute=True')
        if not (np.isscalar(self.noise_min) and np.isscalar(self.noise_max)):
            raise NotImplementedError('GaussianNoise: only scalar noise_min / noise_max are supported')
        seed = None if self.seed is None else self.seed + self._calls
        self._calls += 1
        rand = np.random.default_rng(seed)
        k_sd, k_noise = int(rand.integers(np.iinfo(int).max)), int(rand.integers(np.iinfo(int).max))

        x32 = x if x.dtype == torch.float32 else x.to(torch.float32)
        x32 = x32.contiguous()
        shape_sd = [s if i in self.axes else 1 for i, s in enumerate(x32.shape)]
        n_sd = int(np.prod(shape_sd, dtype=np.int64))
        table = torch.empty(max(n_sd, 1), dtype=torch.float32, device=x.device)
        scale = None
        with torch.cuda.device(x.device):
            st = stream_ptr(x.device)
            check(lib.nrt_philox_uniform_f32(k_sd, n_sd, float(self.noise_min), float(self.noise_max), ptr(table),
                                             st))
            if not self.absolute and x32.numel():
                scale = utils._item_stats(x32.detach().reshape(1, -1), _lib.NRT_STAT_ABSMAX)
        if self.noise_only:
            out = torch.empty_like(x32, memory_format=torch.contiguous_format)
            with torch.cuda.device(x.device):
                check(lib.nrt_philox_normal_f32(k_noise, i32_array(x32.shape), i32_array(shape_sd), x32.dim(),
                                                ptr(table), ptr(scale), None, ptr(out), stream_ptr(x.device)))
        else:
            out = _NoiseAddFn.apply(x32, k_noise, shape_sd, table, scale)
        return out.to(x.dtype) if x.dtype != torch.float32 else out

    def compute_output_shape(self, input_shape):
        return tuple(input_shape)


class PerlinNoise(_Layer):
    """Perlin noise drawn at full resolution for each batch item, reference layers.py:2406-2508: per level an
    SD from U[noise_min, noise_max] (one per index along `axes`), N(0, SD) noise, a random Gaussian blur with
    FWHMs in [fwhm_min, fwhm_max] that keeps `reduce` ('std', 'max' or a callable) constant, and the mean over
    levels.  The input fixes the batch size (and the shape when `shape=None`).  Computed in fp32 and cast to
    `out_type`.  Randomness: see neurite_b200/augment.py; a layer with a seed draws with
    `seed + number of earlier calls`, and every item gets fresh draws."""

    def __init__(self, shape=None, noise_min=0.01, noise_max=1, fwhm_min=4, fwhm_max=32, isotropic=False,
                 reduce='std', out_type=torch.float32, axes=None, seed=None, **kwargs):
        self.shape = shape
        self.noise_min = noise_min
        self.noise_max = noise_max
        self.fwhm_min = fwhm_min
        self.fwhm_max = fwhm_max
        self.isotropic = isotropic
        self.reduce = reduce
        self.out_type = getattr(torch, out_type) if isinstance(out_type, str) else out_type
        self.axes = axes
        self.seed = seed
        self._calls = 0
        super().__init__(**kwargs)

    def get_config(self):
        config = super().get_config().copy()
        config.update({'shape': self.shape, 'noise_min': self.noise_min, 'noise_max': self.noise_max,
                       'fwhm_min': self.fwhm_min, 'fwhm_max': self.fwhm_max, 'isotropic': self.isotropic,
                       'reduce': self.reduce, 'out_type': self.out_type, 'axes': self.axes, 'seed': self.seed})
        return config

    def build(self, input_shape):
        allowed = range(1, len(input_shape))
        self._axes = augment.normalize_axes(self.axes, input_shape, allowed, none_means_all=False)
        super().build(input_shape)

    def _plan(self, x, seed):
        """(per-item level draws, item shape [1, *shape], SD-table shape) of one call with `seed`."""
        fwhm_min, fwhm_max = augment._check_perlin_args(self.noise_min, self.noise_max, self.fwhm_min, self.fwhm_max)
        shape = list(x.shape[1:]) if self.shape is None else [int(s) for s in self.shape]
        gshape = [1] + shape                                   # draw_perlin_full(batched=False, featured=True)
        shape_sd = [gshape[i] if i in self._axes else 1 for i in range(len(gshape))]
        rand = np.random.default_rng(seed)
        draws = [augment._level_draws(np.random.default_rng(int(rand.integers(np.iinfo(int).max))), len(shape) - 1,
                                      fwhm_min, fwhm_max, self.isotropic) for _ in range(x.shape[0])]
        return draws, gshape, shape_sd

    def call(self, x):
        require_cuda(x)
        augment._stat_kind(self.reduce)
        seed = None if self.seed is None else self.seed + self._calls
        self._calls += 1
        draws, gshape, shape_sd = self._plan(x, seed)
        _, fwhm_max = augment._check_perlin_args(self.noise_min, self.noise_max, self.fwhm_min, self.fwhm_max)
        out = augment._perlin(draws, gshape, shape_sd, self.noise_min, self.noise_max, fwhm_max, self.reduce,
                              x.device)
        out = out.reshape([x.shape[0]] + gshape[1:])
        return out.to(self.out_type) if self.out_type != torch.float32 else out

    def compute_output_shape(self, input_shape):
        return (input_shape[0],) + tuple(input_shape[1:] if self.shape is None else self.shape)
