"""
numpy fp32 restatement of soft_quantize and MutualInformation.
TEST INFRASTRUCTURE (see oracle/__init__.py).

Follows adalca/neurite: neurite/tf:
    utils/utils.py:1099-1172  soft_quantize (bin centres default to tf.linspace(min x, max x, nb))
    metrics.py:69-114         MutualInformation.__init__ (alpha = 1 / (2 sigma^2), fp32)
    metrics.py:116-138        volumes          metrics.py:140-152  segs
    metrics.py:154-183        volume_seg       metrics.py:185-225  channelwise
    metrics.py:227-292        maps

Pinned by tests/golden/mi_*.npz (the reference's own source executed on tools/tfshim.py).
Sums (the batched matmul of metrics.py:272 and the K.sum calls) accumulate in float64 and round
once to fp32: TF's reduction order is unspecified, parity tolerance 1e-5.
"""
import numpy as np

from .interp import tf_linspace_f32

F32 = np.float32
EPS = F32(1e-7)          # K.epsilon()


class InvalidArgument(ValueError):
    """Stands in for tf.errors.InvalidArgumentError raised by tf.debugging asserts."""


def soft_quantize(x, bin_centers=None, nb_bins=16, alpha=1, min_clip=-np.inf, max_clip=np.inf,
                  return_log=False):
    """utils.py:1099-1172."""
    x = np.asarray(x, dtype=F32)
    if bin_centers is not None:
        bin_centers = np.asarray(bin_centers, dtype=F32)
        assert nb_bins is None, 'cannot provide both bin_centers and nb_bins'
        nb_bins = bin_centers.shape[0]
    else:
        if nb_bins is None:
            nb_bins = 16
        bin_centers = tf_linspace_f32(np.min(x), np.max(x), nb_bins)              # :1151-1153
    x = np.clip(x[..., None], F32(min_clip), F32(max_clip))                         # :1156-1157
    bin_diff = np.square(x - bin_centers.reshape((1,) * (x.ndim - 1) + (nb_bins,)))  # :1165
    log = -F32(alpha) * bin_diff                                                    # :1166
    return log if return_log else np.exp(log)


def default_alpha(nb_bins=None, bin_centers=None):
    """metrics.py:105-113: sigma = 0.5 / (nb - 1) or 0.5 * mean(diff(centers)); alpha = 1 / (2 * square(sigma)),
    the square, the product and the reciprocal in fp32 (tf.square of a python float is an fp32 tensor)."""
    if bin_centers is None:
        sigma = F32(0.5 / (nb_bins - 1))
    else:
        sigma = F32(0.5) * F32(np.mean(np.diff(np.asarray(bin_centers, dtype=F32)), dtype=np.float64))
    return F32(1) / (F32(2) * (sigma * sigma))


class MutualInformation:
    def __init__(self, bin_centers=None, nb_bins=None, soft_bin_alpha=None, min_clip=None, max_clip=None):
        self.bin_centers = None
        if bin_centers is not None:
            self.bin_centers = np.asarray(bin_centers, dtype=F32)
            assert nb_bins is None, 'cannot provide both bin_centers and nb_bins'
            nb_bins = self.bin_centers.shape[0]
        self.nb_bins = nb_bins
        if bin_centers is None and nb_bins is None:
            self.nb_bins = 16
        self.min_clip = -np.inf if min_clip is None else min_clip
        self.max_clip = np.inf if max_clip is None else max_clip
        self.soft_bin_alpha = soft_bin_alpha
        if self.soft_bin_alpha is None:
            self.soft_bin_alpha = default_alpha(self.nb_bins, self.bin_centers)

    def _soft_sim_map(self, x):                                                     # :320-336
        # (soft_quantize asserts nb_bins is None when centres are given; the reference passes both
        #  -- metrics.py:329-331 -- and would trip that assert, so centres imply nb_bins=None here)
        return soft_quantize(x, alpha=self.soft_bin_alpha, bin_centers=self.bin_centers,
                             nb_bins=None if self.bin_centers is not None else self.nb_bins,
                             min_clip=self.min_clip, max_clip=self.max_clip, return_log=False)

    def volumes(self, x, y):                                                        # :116-138
        x, y = np.asarray(x, F32), np.asarray(y, F32)
        if x.shape[-1] != 1 or y.shape[-1] != 1:
            raise InvalidArgument('volume_mi requires two single-channel volumes. See channelwise().')
        return self.channelwise(x, y).reshape(-1)

    def segs(self, x, y):                                                           # :140-152
        return self.maps(x, y)

    def volume_seg(self, x, y):                                                     # :154-183
        x, y = np.asarray(x, F32), np.asarray(y, F32)
        cx, cy = x.shape[-1], y.shape[-1]
        if min(cx, cy) != 1:
            raise InvalidArgument('volume_seg_mi requires one single-channel volume.')
        if not max(cx, cy) > 1:
            raise InvalidArgument('volume_seg_mi requires one multi-channel segmentation.')
        if cx == 1:
            x = self._soft_sim_map(x[..., 0])
        else:
            y = self._soft_sim_map(y[..., 0])
        return self.maps(x, y)

    def channelwise(self, x, y):                                                    # :185-225
        x, y = np.asarray(x, F32), np.asarray(y, F32)
        if x.shape != y.shape:
            raise InvalidArgument('volume shapes do not match')
        if x.ndim != 3:
            x = x.reshape(x.shape[0], -1, x.shape[-1])
            y = y.reshape(y.shape[0], -1, y.shape[-1])
        cx = np.moveaxis(x, -1, 0)                                                  # [C, bs, V]
        cy = np.moveaxis(y, -1, 0)
        cxq = self._soft_sim_map(cx)                                                # min/max over ALL of cx
        cyq = self._soft_sim_map(cy)
        out = np.stack([self.maps(a, b) for a, b in zip(cxq, cyq)], 0)              # [C, bs]
        return out.T

    def maps(self, x, y):                                                           # :227-292
        x, y = np.asarray(x, F32), np.asarray(y, F32)
        if x.shape != y.shape:
            raise InvalidArgument('shapes %s and %s differ' % (x.shape, y.shape))   # :261
        if not np.all(x >= 0) or not np.all(y >= 0):
            raise InvalidArgument('negative value')                                 # :262-263
        if x.ndim != 3:
            x = x.reshape(x.shape[0], -1, x.shape[-1])
            y = y.reshape(y.shape[0], -1, y.shape[-1])
        x64, y64 = x.astype(np.float64), y.astype(np.float64)
        pxy = np.einsum('bvi,bvj->bij', x64, y64).astype(F32)                       # :271-272
        pxy = pxy / (np.sum(pxy, axis=(1, 2), keepdims=True, dtype=np.float64).astype(F32) + EPS)
        px = np.sum(x64, 1, keepdims=True).astype(F32)                              # :276
        px = px / (np.sum(px, 2, keepdims=True, dtype=np.float64).astype(F32) + EPS)
        py = np.sum(y64, 1, keepdims=True).astype(F32)
        py = py / (np.sum(py, 2, keepdims=True, dtype=np.float64).astype(F32) + EPS)
        pxpy = np.transpose(px, (0, 2, 1)) * py                                     # [bs,B1,1] x [bs,1,B2]
        pxpy_eps = pxpy + EPS
        log_term = np.log(pxy / pxpy_eps + EPS)                                     # :290
        return np.sum(pxy * log_term, axis=(1, 2), dtype=np.float64).astype(F32)    # :291


# ---------------------------------------------------------------------------------------
# differentiable float64 restatement (torch autograd on the CPU): the gradient oracle.
# TF differentiates the same graph -- clip_by_value passes the gradient on the closed interval,
# reduce_min / reduce_max send it to the extremal elements (shared evenly among ties), and the
# linspace centres carry it to min and max.
# ---------------------------------------------------------------------------------------
def torch_soft_quantize(x, nb_bins=None, alpha=1.0, min_clip=-np.inf, max_clip=np.inf, bin_centers=None):
    import torch
    if bin_centers is None:
        mn, mx = x.min(), x.max()
        i = torch.arange(nb_bins, dtype=x.dtype)
        centers = mn + (mx - mn) / (nb_bins - 1) * i if nb_bins > 1 else mn.reshape(1)
    else:
        centers = torch.as_tensor(np.asarray(bin_centers), dtype=x.dtype)
    xc = torch.clamp(x[..., None], min_clip, max_clip)
    return torch.exp(-alpha * (xc - centers) ** 2)


def torch_maps(x, y):
    import torch
    eps = 1e-7
    x = x.reshape(x.shape[0], -1, x.shape[-1])
    y = y.reshape(y.shape[0], -1, y.shape[-1])
    pxy = torch.einsum('bvi,bvj->bij', x, y)
    pxy = pxy / (pxy.sum(dim=(1, 2), keepdim=True) + eps)
    px = x.sum(1, keepdim=True)
    px = px / (px.sum(2, keepdim=True) + eps)
    py = y.sum(1, keepdim=True)
    py = py / (py.sum(2, keepdim=True) + eps)
    pxpy = px.transpose(1, 2) * py
    return (pxy * torch.log(pxy / (pxpy + eps) + eps)).sum(dim=(1, 2))


def torch_channelwise(x, y, nb_bins=16, alpha=None, min_clip=-np.inf, max_clip=np.inf, bin_centers=None):
    """x, y: torch float64 [bs, ..., C] -> [bs, C] (metrics.py:185-225)."""
    import torch
    if alpha is None:
        alpha = float(default_alpha(nb_bins, bin_centers))
    x = x.reshape(x.shape[0], -1, x.shape[-1])
    y = y.reshape(y.shape[0], -1, y.shape[-1])
    cxq = torch_soft_quantize(x.permute(2, 0, 1), nb_bins, alpha, min_clip, max_clip, bin_centers)   # [C, bs, V, B]
    cyq = torch_soft_quantize(y.permute(2, 0, 1), nb_bins, alpha, min_clip, max_clip, bin_centers)
    return torch.stack([torch_maps(a, b) for a, b in zip(cxq, cyq)], 0).T


def torch_volume_seg(vol, seg, nb_bins=16, alpha=None, min_clip=-np.inf, max_clip=np.inf):
    if alpha is None:
        alpha = float(default_alpha(nb_bins, None))
    return torch_maps(torch_soft_quantize(vol[..., 0], nb_bins, alpha, min_clip, max_clip), seg)
