"""
numpy restatement of gaussian_kernel / separable_conv / GaussianBlur / subsample_axis.
TEST INFRASTRUCTURE (see oracle/__init__.py).

Follows adalca/neurite: neurite/tf:
    utils/utils.py:581-662   gaussian_kernel
    utils/utils.py:665-751   separable_conv   (tf.nn.convolution: third party, TF unpinned --
                             cross-correlation, 'SAME' = zero padding with the extra element at
                             the end, out = ceil(in / stride); 'VALID' = ceil((in - (k-1)d) / stride))
    layers.py:251-364        GaussianBlur
    utils/utils.py:754-826   subsample_axis   (the random draws are arguments here)

Pinned by tests/golden/blur_*.npz / gausskernel_*.npz: the reference's own source executed on
tools/tfshim.py, whose tf.nn.convolution is this file's `conv1d_axis` (contract, not reference
code).  Tap sums accumulate in float64 and round once (TF's order is unspecified).
"""
import numpy as np

from .interp import tf_linspace_f32

F32 = np.float32


def gaussian_kernel(sigma, windowsize=None, indexing='ij', separate=False):
    """utils.py:581-662 without the random branch (sigma drawn by the caller)."""
    if not isinstance(sigma, (list, tuple)):
        sigma = [sigma]
    eps = np.finfo(np.float32).eps
    sigma = [max(f, eps) for f in sigma]                                            # :628
    if windowsize is None:
        windowsize = [np.round(f * 3) * 2 + 1 for f in sigma]                       # :633
    if not isinstance(windowsize, (list, tuple)):
        windowsize = [windowsize]
    if len(sigma) != len(windowsize):
        raise ValueError(f'sigma {sigma} and width {windowsize} differ in length')
    center = [(w - 1) / 2 for w in windowsize]
    mesh = [np.arange(w) - c for w, c in zip(windowsize, center)]
    mesh = [-0.5 * x**2 for x in mesh]                                              # float64
    if not separate:
        mesh = np.meshgrid(*mesh, indexing=indexing)
    mesh = [m.astype(F32) for m in mesh]                                            # tf.constant(m, fp32)
    exponent = [m / F32(s**2) for m, s in zip(mesh, sigma)]                         # :654, fp32 divide
    if not separate:
        exponent = [np.sum(np.stack(exponent), axis=0, dtype=np.float64).astype(F32)]
    kernel = [np.exp(x) for x in exponent]
    kernel = [x / np.sum(x, dtype=np.float64).astype(F32) for x in kernel]
    return kernel if len(kernel) > 1 else kernel[0]


def same_padding(n, k, stride=1, dilation=1):
    """TF 'SAME': (n_out, pad_before)."""
    n_out = -(-n // stride)
    eff = (k - 1) * dilation + 1
    total = max((n_out - 1) * stride + eff - n, 0)
    return n_out, total // 2


def conv1d_axis(x, k, axis, padding='SAME', stride=1, dilation=1):
    """Cross-correlate every 1-D line of x along `axis` with k (tf.nn.convolution with a kernel
    that is 1 everywhere but along that axis, one input and one output feature)."""
    x = np.asarray(x, F32)
    k = np.asarray(k, F32).ravel()
    n, K = x.shape[axis], k.shape[0]
    if stride > 1 and dilation > 1:
        raise ValueError('strides > 1 not supported in conjunction with dilation_rate > 1')
    if padding.upper() == 'SAME':
        n_out, pb = same_padding(n, K, stride, dilation)
    else:
        n_out, pb = max(-(-(n - (K - 1) * dilation) // stride), 0), 0
    xm = np.moveaxis(x, axis, 0).astype(np.float64)
    out = np.zeros((n_out,) + xm.shape[1:], np.float64)
    for o in range(n_out):
        for j in range(K):
            s = o * stride - pb + j * dilation
            if 0 <= s < n:
                out[o] += np.float64(k[j]) * xm[s]
    return np.moveaxis(out.astype(F32), 0, axis)


def separable_conv(x, kernels, axis=None, batched=False, padding='SAME', strides=None, dilations=None):
    """utils.py:665-751 ([..., C] trailing feature dimension; the same filters across features)."""
    x = np.asarray(x, F32)
    if not batched:
        x = x[None]
    num_dim = x.ndim - 2
    if np.isscalar(axis):
        axis = [axis]
    if axis is None:
        axis = list(range(num_dim))
    assert all(ax in range(num_dim) for ax in axis), 'non-spatial axis passed'
    def conform(v):
        v = np.ravel(1 if v is None else v).tolist()
        return v * len(axis) if len(v) == 1 else v
    strides, dilations = conform(strides), conform(dilations)
    assert len(strides) == len(axis), 'number of strides and axes differ'
    assert len(dilations) == len(axis), 'number of dilations and axes differ'
    if not isinstance(kernels, (tuple, list)):
        kernels = [kernels]
    if len(kernels) == 1:
        kernels = list(kernels) * len(axis)
    assert len(kernels) == len(axis), 'number of kernels and axes differ'
    for ax, k, s, d in zip(axis, kernels, strides, dilations):
        x = conv1d_axis(x, k, ax + 1, padding, int(s), int(d))
    return x if batched else x[0]


def gaussian_blur(x, sigma):
    """layers.py:251-364 GaussianBlur(sigma)(x), non-random: x [B, *space, C]."""
    x = np.asarray(x, F32)
    ndims = x.ndim - 2
    sigma = np.ravel(sigma).tolist()
    if len(sigma) not in (1, ndims):
        raise ValueError(f'1 or {ndims} sigmas expected in {ndims}D space, got {len(sigma)}')
    if any(s < 0 for s in sigma):
        raise ValueError('Gaussian blur sigma must not be less than 0')
    if len(sigma) == 1:
        sigma = sigma * ndims
    if not any(s > 0 for s in sigma):
        return x
    kernel = gaussian_kernel(sigma, separate=True)
    if ndims == 1:
        kernel = [kernel]
    return separable_conv(x, list(kernel), batched=True)


def subsample_indices(width, thick, upsample=True):
    """utils.py:812-823: the gather indices for a drawn thickness (fp32 arithmetic)."""
    num_slice = int(F32(width) / F32(thick) + F32(0.5))
    ind = (tf_linspace_f32(0, width - 1, num_slice) + F32(0.5)).astype(np.int32)
    if not upsample:
        return ind
    up = (tf_linspace_f32(0, num_slice - 1, width) + F32(0.5)).astype(np.int32)
    return ind[up]


def subsample_axis(x, ax, thick, upsample=True):
    x = np.asarray(x)
    return np.take(x, subsample_indices(x.shape[ax], thick, upsample), axis=ax)
