"""
numpy fp32 restatement of LocallyConnected3D, implementation 1.  TEST INFRASTRUCTURE
(see oracle/__init__.py).

Follows adalca/neurite: neurite/tf/layers.py:
    build (shapes)            :951-1047
    call (bias, activation)   :1072-1102
    local_conv (impl 1)       :1126-1197
    conv_kernel_idxs docstring known answer :1354-1363
"""
import itertools

import numpy as np

F32 = np.float32


def conv_output_length(input_length, filter_size, padding, stride):
    """keras conv_utils.conv_output_length ('valid' / 'same'), used at layers.py:963-968."""
    if input_length is None:
        return None
    assert padding in ('valid', 'same')
    if padding == 'same':
        out = input_length
    else:
        out = input_length - filter_size + 1
    return (out + stride - 1) // stride


def output_shape(in_spatial, kernel_size, strides, padding='valid'):
    return tuple(conv_output_length(in_spatial[d], kernel_size[d], padding, strides[d]) for d in range(3))


def local_conv(inputs, kernel, kernel_size, strides, out_shape, data_format='channels_last'):
    """layers.py:1126-1197, literally: one slice+reshape per output position (python loop),
    concatenate to [P, B, F], batched dot with kernel [P, F, Cout], reshape, permute.
    Only usable for small P (the reference builds P graph ops the same way)."""
    if data_format not in {'channels_first', 'channels_last'}:
        raise ValueError('Unknown data_format: ' + str(data_format))
    inputs = np.asarray(inputs, dtype=F32)
    kernel = np.asarray(kernel, dtype=F32)
    feature_dim = kernel.shape[1]
    channels_out = kernel.shape[-1]
    ndims = len(out_shape)
    spatial_dimensions = list(range(ndims))

    xs = []
    for position in itertools.product(*[range(m) for m in out_shape]):          # :1172-1173
        slices = [slice(None)]
        if data_format == 'channels_first':
            slices.append(slice(None))
        slices.extend([slice(position[d] * strides[d], position[d] * strides[d] + kernel_size[d])
                       for d in spatial_dimensions])                            # :1179-1181
        if data_format == 'channels_last':
            slices.append(slice(None))
        xs.append(np.reshape(inputs[tuple(slices)], (1, -1, feature_dim)))      # :1186
    x_aggregate = np.concatenate(xs, axis=0)                                    # :1188  [P,B,F]
    output = np.matmul(x_aggregate, kernel)                                     # :1189  K.batch_dot
    output = np.reshape(output, tuple(out_shape) + (-1, channels_out))          # :1190
    if data_format == 'channels_first':
        permutation = [ndims, ndims + 1] + spatial_dimensions
    else:
        permutation = [ndims] + spatial_dimensions + [ndims + 1]
    return np.transpose(output, permutation)                                    # :1197


def local_conv_fast(inputs, kernel, kernel_size, strides, out_shape, data_format='channels_last'):
    """Loop-free equivalent of local_conv (strided window view + einsum) for sizes where
    the literal P-iteration loop is impractical.  Same patch-feature ordering
    j = ((i0*k1+i1)*k2+i2)*Cin + c (channels_last) / ((c*k0+i0)*k1+i1)*k2+i2 (channels_first)."""
    inputs = np.asarray(inputs, dtype=F32)
    kernel = np.asarray(kernel, dtype=F32)
    k0, k1, k2 = kernel_size
    s0, s1, s2 = strides
    o0, o1, o2 = out_shape
    cout = kernel.shape[-1]
    if data_format == 'channels_first':
        x = np.moveaxis(inputs, 1, -1)
    else:
        x = inputs
    B, _, _, _, cin = x.shape
    from numpy.lib.stride_tricks import as_strided
    st = x.strides
    win = as_strided(x, shape=(B, o0, o1, o2, k0, k1, k2, cin),
                     strides=(st[0], st[1] * s0, st[2] * s1, st[3] * s2, st[1], st[2], st[3], st[4]),
                     writeable=False)
    if data_format == 'channels_first':
        kr = kernel.reshape(o0, o1, o2, cin, k0, k1, k2, cout)
        out = np.einsum('bxyzijkc,xyzcijkf->bxyzf', win, kr, optimize=True)
        return np.ascontiguousarray(np.moveaxis(out, -1, 1)).astype(F32)
    kr = kernel.reshape(o0, o1, o2, k0, k1, k2, cin, cout)
    out = np.einsum('bxyzijkc,xyzijkcf->bxyzf', win, kr, optimize=True)
    return out.astype(F32)


_ACTIVATIONS = {
    None: lambda v: v,
    'linear': lambda v: v,
    'relu': lambda v: np.maximum(v, F32(0)),
    'sigmoid': lambda v: (F32(1) / (F32(1) + np.exp(-v))).astype(F32),
    'tanh': lambda v: np.tanh(v).astype(F32),
}


def locally_connected_3d(inputs, kernel, bias, kernel_size, strides=(1, 1, 1), padding='valid',
                         data_format='channels_last', activation=None, literal=None):
    """LocallyConnected3D.call for implementation 1 (layers.py:1072-1102): local_conv, then
    K.bias_add with bias [o0,o1,o2,Cout] (:1034-1040, :1098-1099), then activation (:1101)."""
    if padding != 'valid':
        raise ValueError('Invalid border mode for LocallyConnected3D '
                         '(only "valid" is supported if implementation is 1): ' + padding)
    inputs = np.asarray(inputs, dtype=F32)
    spatial = inputs.shape[1:4] if data_format == 'channels_last' else inputs.shape[2:5]
    out_shape = output_shape(spatial, kernel_size, strides, padding)
    P = int(np.prod(out_shape))
    if literal is None:
        literal = P <= 4096
    fn = local_conv if literal else local_conv_fast
    out = fn(inputs, kernel, kernel_size, strides, out_shape, data_format)
    if bias is not None:
        bias = np.asarray(bias, dtype=F32)
        if data_format == 'channels_first':
            # K.bias_add(channels_first) with a [o0,o1,o2,C] bias: raw reshape to (1, C, o0, o1, o2), not a transpose
            out = out + bias.reshape((bias.shape[-1],) + bias.shape[:-1])[None]
        else:
            out = out + bias[None]
    return _ACTIVATIONS[activation](out).astype(F32)
