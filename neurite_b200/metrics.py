"""
neurite_b200.metrics -- drop-ins for Dice / SoftDice / HardDice / CategoricalCrossentropy of
neurite.metrics (adalca/neurite: neurite/tf/metrics.py:339-650) on torch CUDA tensors.

Same constructor arguments, defaults, assertions and method names (`dice`, `mean_dice`,
`loss`, `cce`, `__call__`).  tf.debugging asserts become `InvalidArgumentError`
(a ValueError) carrying the reference's messages 'value outside range' / 'metric not finite'.

`group`, when given, is a torch.distributed process group over which the voxel range of
every batch item is sharded: each rank passes its own voxel slab and the [B,L,3] partial
sums (768 B at cfg 3) are all-reduced before the finalize kernel (SURVEY.md 8e).
"""
import warnings

import numpy as np
import torch

from . import utils
from ._lib import lib, check, ptr, stream_ptr, require_cuda


class InvalidArgumentError(ValueError):
    """Raised where the reference's tf.debugging asserts raise tf.errors.InvalidArgumentError."""


_WS = {}
_WS_MAX_STREAMS = 8


def _workspace(device, nbytes):
    """Per (device, stream) scratch for the block partials of the reductions (1.6 MB at
    cfg 3): launches on the same stream are ordered, so one buffer per stream is race free.
    The cache is bounded: beyond _WS_MAX_STREAMS streams the oldest entry is dropped (the caching allocator keeps
    its memory alive for the kernels already queued on that stream), so short-lived streams do not leak buffers."""
    return utils._stream_scratch(_WS, _WS_MAX_STREAMS, device, nbytes)


def dice_sums(y_true, y_pred, normalize=False, check_input_limits=True, group=None):
    """[B,*S,L] x2 -> sums [B,L,3] = (sum t*p, sum t*t, sum p*p) and a range flag tensor."""
    require_cuda(y_true, y_pred)
    if y_true.shape != y_pred.shape:
        raise ValueError('y_true %s and y_pred %s differ in shape' % (tuple(y_true.shape), tuple(y_pred.shape)))
    t = y_true.to(torch.float32).contiguous()
    p = y_pred.to(torch.float32).contiguous()
    B, L = t.shape[0], t.shape[-1]
    V = t.numel() // max(B * L, 1)
    sums = torch.empty((B, L, 3), dtype=torch.float32, device=t.device)
    flag = torch.zeros(1, dtype=torch.int32, device=t.device)
    ws_bytes = lib.nrt_dice_workspace_bytes(B, L)
    ws = _workspace(t.device, ws_bytes)
    with torch.cuda.device(t.device):
        check(lib.nrt_dice_sums_f32(ptr(t), ptr(p), B, V, L, 0, V, int(bool(normalize)), int(bool(check_input_limits)),
                                    ptr(sums), ptr(flag), ptr(ws), ws_bytes, stream_ptr(t.device)))
    if group is not None:
        # one collective: the [B,L,3] partial sums and the range flag travel together
        import torch.distributed as dist
        packed = torch.cat([sums.reshape(-1), flag.to(torch.float32)])
        dist.all_reduce(packed, group=group)
        sums = packed[:-1].reshape(B, L, 3).contiguous()
        flag = (packed[-1:] > 0).to(torch.int32)
    return sums, flag


def dice_label_sums(t_lab, p_lab, nb_labels, group=None):
    """integer label maps [B,*S] x2 -> sums [B,L,3] (exact counts)."""
    require_cuda(t_lab, p_lab)
    t = t_lab.to(torch.int32).contiguous()
    p = p_lab.to(torch.int32).contiguous()
    B = t.shape[0]
    V = t.numel() // max(B, 1)
    sums = torch.empty((B, nb_labels, 3), dtype=torch.float32, device=t.device)
    ws_bytes = lib.nrt_dice_workspace_bytes(B, nb_labels)
    ws = _workspace(t.device, ws_bytes)
    with torch.cuda.device(t.device):
        check(lib.nrt_dice_label_sums_i32(ptr(t), ptr(p), B, V, nb_labels, 0, V, ptr(sums), ptr(ws), ws_bytes,
                                          stream_ptr(t.device)))
    if group is not None:
        import torch.distributed as dist
        dist.all_reduce(sums, group=group)
    return sums


def argmax_labels(x):
    """[..., L] float -> [...] int32, first maximum wins (tf.argmax)."""
    require_cuda(x)
    x32 = x.to(torch.float32).contiguous()
    L = x32.shape[-1]
    n = x32.numel() // L
    idx = torch.empty(x32.shape[:-1], dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.nrt_argmax_f32(ptr(x32), n, L, ptr(idx), stream_ptr(x.device)))
    return idx


def dice_finalize(sums, laplace_smoothing=0.):
    B, L = sums.shape[0], sums.shape[1]
    out = torch.empty((B, L), dtype=torch.float32, device=sums.device)
    with torch.cuda.device(sums.device):
        check(lib.nrt_dice_finalize_f32(ptr(sums), B, L, float(laplace_smoothing), ptr(out), stream_ptr(sums.device)))
    return out


class _DiceFn(torch.autograd.Function):
    """autograd shell: nrt_dice_sums_f32 + nrt_dice_finalize_f32 forward, nrt_dice_bwd_f32 backward."""

    @staticmethod
    def forward(ctx, y_true, y_pred, check, laplace):
        t = y_true.detach().to(torch.float32).contiguous()
        p = y_pred.detach().to(torch.float32).contiguous()
        sums, flag = dice_sums(t, p, False, check, None)
        if check and int(flag.item()) != 0:
            raise InvalidArgumentError('value outside range')
        ctx.save_for_backward(t, p, sums)
        ctx.laplace = laplace
        return dice_finalize(sums, laplace)

    @staticmethod
    def backward(ctx, g):
        t, p, sums = ctx.saved_tensors
        g = g.contiguous().to(torch.float32)
        B, L = sums.shape[0], sums.shape[1]
        V = t.numel() // max(B * L, 1)
        gt = torch.empty_like(t) if ctx.needs_input_grad[0] else None
        gp = torch.empty_like(p) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(t.device):
            check(lib.nrt_dice_bwd_f32(ptr(t), ptr(p), ptr(sums), ptr(g), B, V, L, ctx.laplace, ptr(gt), ptr(gp),
                                       stream_ptr(t.device)))
        return gt, gp, None, None


class _CceFn(torch.autograd.Function):
    """autograd shell: nrt_cce_f32 forward, nrt_cce_bwd_f32 backward (gradient wrt y_pred)."""

    @staticmethod
    def forward(ctx, t, p, lw, sw, from_logits, smoothing, reduction):
        C = p.shape[-1]
        n = p.numel() // C
        per = torch.empty(p.shape[:-1], dtype=torch.float32, device=p.device) if reduction == 'none' else None
        total = torch.empty(1, dtype=torch.float32, device=p.device)
        ws_bytes = lib.nrt_cce_workspace_bytes()
        ws = _workspace(p.device, ws_bytes)
        with torch.cuda.device(p.device):
            check(lib.nrt_cce_f32(ptr(t), ptr(p), ptr(lw), ptr(sw), n, C, int(from_logits), float(smoothing),
                                  ptr(per), ptr(total), ptr(ws), ws_bytes, stream_ptr(p.device)))
        ctx.save_for_backward(t, p, lw, sw)
        ctx.args = (from_logits, smoothing, reduction, n, C)
        if reduction == 'none':
            return per
        return total[0] if reduction == 'sum' else total[0] / n

    @staticmethod
    def backward(ctx, g):
        t, p, lw, sw = ctx.saved_tensors
        from_logits, smoothing, reduction, n, C = ctx.args
        g = g.contiguous().to(torch.float32)
        gp = torch.empty_like(p)
        gper = g if reduction == 'none' else None
        gscal = g.reshape(1) if reduction != 'none' else None
        scale = 1.0 / n if reduction == 'sum_over_batch_size' else 1.0
        with torch.cuda.device(p.device):
            check(lib.nrt_cce_bwd_f32(ptr(t), ptr(p), ptr(lw), ptr(sw), n, C, int(from_logits), float(smoothing),
                                      ptr(gscal), scale, ptr(gper), ptr(gp), stream_ptr(p.device)))
        return None, gp, None, None, None, None, None


class Dice:
    """Dice of two Tensors -- reference metrics.py:339-519."""

    def __init__(self, dice_type='soft', input_type='prob', nb_labels=None, weights=None,
                 check_input_limits=True, laplace_smoothing=0., normalize=False, group=None):
        self.dice_type = dice_type
        self.input_type = input_type
        self.nb_labels = nb_labels
        self.weights = weights
        self.normalize = normalize
        self.check_input_limits = check_input_limits
        self.laplace_smoothing = laplace_smoothing
        self.group = group
        assert self.input_type in ['prob', 'max_label']                                   # :406
        if self.dice_type == 'hard' and self.input_type == 'max_label':
            assert self.nb_labels is not None, 'If doing hard Dice need nb_labels'       # :408-409
        if self.dice_type == 'soft':
            assert self.input_type in ['prob', 'one_hot'], \
                'if doing soft Dice, must use probabilistic (one_hot)encoding'           # :411-413

    def dice(self, y_true, y_pred):
        """[batch, ..., nb_labels] (prob) or [batch, ...] (max_label) -> [batch, nb_labels]."""
        if self.dice_type == 'hard':
            if self.input_type == 'prob':
                warnings.warn('You are using ne.metrics.Dice with probabilistic inputs'
                              'and computing *hard* dice. \n For this, we use argmax to'
                              'get the optimal label at each location, which is not'
                              'differentiable. Do not use expecting gradients.')          # :455-458
                if self.check_input_limits or self.normalize:
                    # the reference checks / renormalises the probabilistic inputs first (:434-444)
                    _, flag = dice_sums(y_true, y_pred, self.normalize, self.check_input_limits, self.group)
                    if self.check_input_limits and int(flag.item()) != 0:
                        raise InvalidArgumentError('value outside range')
                if self.nb_labels is None:
                    self.nb_labels = int(y_pred.shape[-1])                                # :460-461
                y_pred = argmax_labels(y_pred)                                            # :463-464
                y_true = argmax_labels(y_true)
            sums = dice_label_sums(y_true, y_pred, self.nb_labels, self.group)           # :467-477 fused
        else:
            needs_grad = torch.is_grad_enabled() and (y_pred.requires_grad or y_true.requires_grad)
            if needs_grad:
                if self.normalize or self.group is not None:
                    raise NotImplementedError('Dice gradients are built for normalize=False on one device')
                return _DiceFn.apply(y_true, y_pred, bool(self.check_input_limits), float(self.laplace_smoothing))
            sums, flag = dice_sums(y_true, y_pred, self.normalize, self.check_input_limits, self.group)
            if self.check_input_limits and int(flag.item()) != 0:                         # :439-444
                raise InvalidArgumentError('value outside range')
        return dice_finalize(sums, self.laplace_smoothing)                                # :476-482

    def mean_dice(self, y_true, y_pred):
        dice_metric = self.dice(y_true, y_pred)                                           # :499
        if self.weights is not None:                                                      # :502-505
            w = self.weights
            assert len(w.shape) == 2, \
                'weights should be a matrix broadcastable to [batch_size, nb_labels]'
            w = torch.as_tensor(np.asarray(w) if not torch.is_tensor(w) else w, dtype=torch.float32,
                                device=dice_metric.device)
            dice_metric = dice_metric * w
        mean_dice_metric = dice_metric.mean()                                             # :508
        if not bool(torch.isfinite(mean_dice_metric)):
            raise InvalidArgumentError('metric not finite')                               # :509
        return mean_dice_metric

    def loss(self, y_true, y_pred):
        """deprecated alias kept by the reference (metrics.py:512-519)."""
        warnings.warn('ne.metrics.*.loss functions are deprecated.'
                      'Please use the ne.losses.*.loss functions.')
        return -self.mean_dice(y_true, y_pred)


class SoftDice(Dice):
    """reference metrics.py:522-560."""

    def __init__(self, weights=None, check_input_limits=True, laplace_smoothing=0., normalize=False, group=None):
        super().__init__(dice_type='soft', input_type='prob', weights=weights,
                         check_input_limits=check_input_limits, laplace_smoothing=laplace_smoothing,
                         normalize=normalize, group=group)


class HardDice(Dice):
    """reference metrics.py:563-616."""

    def __init__(self, nb_labels, input_type='max_label', weights=None, check_input_limits=True,
                 laplace_smoothing=0., normalize=False, group=None):
        super().__init__(dice_type='hard', input_type=input_type, nb_labels=nb_labels, weights=weights,
                         check_input_limits=check_input_limits, laplace_smoothing=laplace_smoothing,
                         normalize=normalize, group=group)


class CategoricalCrossentropy:
    """Label-weighted categorical cross-entropy -- reference metrics.py:619-650 wrapping
    tf.keras.losses.CategoricalCrossentropy (kwargs from_logits, label_smoothing, axis,
    reduction pass through; axis must be -1)."""

    def __init__(self, label_weights=None, from_logits=False, label_smoothing=0., axis=-1,
                 reduction='sum_over_batch_size', name='categorical_crossentropy', group=None):
        self.label_weights = None
        if label_weights is not None:
            self.label_weights = torch.as_tensor(np.asarray(label_weights) if not torch.is_tensor(label_weights)
                                                 else label_weights)
        if axis != -1:
            raise NotImplementedError('CategoricalCrossentropy: only axis=-1 (channels-last) is built')
        if reduction in ('auto', 'sum_over_batch_size'):
            reduction = 'sum_over_batch_size'
        if reduction not in ('sum_over_batch_size', 'sum', 'none'):
            raise ValueError('Invalid Reduction Key: %s' % reduction)
        self.from_logits = from_logits
        self.label_smoothing = label_smoothing
        self.reduction = reduction
        self.name = name
        self.group = group

    def __call__(self, y_true, y_pred, sample_weight=None):
        return self.cce(y_true, y_pred, sample_weight=sample_weight)

    def cce(self, y_true, y_pred, sample_weight=None):
        lw = None
        if self.label_weights is not None:
            yf = y_pred.shape[-1]
            lf = self.label_weights.shape[-1]
            if yf != lf:
                raise ValueError(f'Label weights must be of len {yf}, but got {lf}.')     # :642-645
            lw = self.label_weights.to(device=y_pred.device, dtype=torch.float32).contiguous()
        require_cuda(y_true, y_pred)
        t = y_true.to(torch.float32).contiguous()
        p = y_pred.to(torch.float32).contiguous()
        C = p.shape[-1]
        n = p.numel() // C
        sw = None
        if sample_weight is not None:
            sw = torch.as_tensor(sample_weight, dtype=torch.float32, device=p.device)
            sw = sw.expand(p.shape[:-1]).contiguous() if sw.dim() > 0 else sw.expand(p.shape[:-1]).contiguous()
        if torch.is_grad_enabled() and y_true.requires_grad:
            # TF autodiff would return dL/dy_true (soft / learned targets); that gradient is not built here and must
            # not be dropped silently
            raise NotImplementedError('CategoricalCrossentropy: gradients w.r.t. y_true are not implemented '
                                      '(detach the target, or use a differentiable torch expression for it)')
        if torch.is_grad_enabled() and y_pred.requires_grad:
            if self.group is not None:
                raise NotImplementedError('CCE gradients are built for one device')
            return _CceFn.apply(t, p, lw, sw, bool(self.from_logits), float(self.label_smoothing), self.reduction)
        per = torch.empty(p.shape[:-1], dtype=torch.float32, device=p.device) if self.reduction == 'none' else None
        total = torch.empty(1, dtype=torch.float32, device=p.device)
        ws_bytes = lib.nrt_cce_workspace_bytes()
        ws = _workspace(p.device, ws_bytes)
        with torch.cuda.device(p.device):
            check(lib.nrt_cce_f32(ptr(t), ptr(p), ptr(lw), ptr(sw), n, C, int(bool(self.from_logits)),
                                  float(self.label_smoothing), ptr(per), ptr(total), ptr(ws), ws_bytes,
                                  stream_ptr(p.device)))
        if self.reduction == 'none':
            return per
        count = torch.tensor([float(n)], device=p.device)
        if self.group is not None:
            import torch.distributed as dist
            dist.all_reduce(total, group=self.group)
            dist.all_reduce(count, group=self.group)
        if self.reduction == 'sum':
            return total[0]
        return (total / count)[0]


class _MiFn(torch.autograd.Function):
    """autograd shell of the mutual information of two operands [B, nv, stride]:
    forward  = (min/max -> centres) + nrt_mi_hist_f32 + nrt_mi_finalize_f32,
    backward = nrt_mi_finalize_bwd_f32 + nrt_mi_bwd_f32 (+ nrt_mi_minmax_bwd_f32 for the centres)."""

    @staticmethod
    def forward(ctx, x, y, mi, xq, yq, nbx, nby, B, C, nv):
        x, y = x.detach(), y.detach()
        dev = x.device
        mmx = mi._range(x) if xq else None
        mmy = mi._range(y) if yq else None
        cx = mi._centers(x, mmx) if xq else None
        cy = mi._centers(y, mmy) if yq else None
        items = B * C
        stats = torch.empty((items, nbx * nby + nbx + nby), dtype=torch.float32, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        ws_bytes = lib.nrt_mi_workspace_bytes(items, nbx, nby)
        ws = _workspace(dev, ws_bytes)
        with torch.cuda.device(dev):
            check(lib.nrt_mi_hist_f32(ptr(x), nv * x.shape[-1], x.shape[-1], int(xq), nbx, ptr(cx),
                                      ptr(y), nv * y.shape[-1], y.shape[-1], int(yq), nby, ptr(cy),
                                      B, C, nv, float(mi.soft_bin_alpha), float(mi.min_clip),
                                      float(mi.max_clip), ptr(stats), ptr(flag), ptr(ws), ws_bytes, stream_ptr(dev)))
        if mi.group is not None:
            import torch.distributed as dist
            packed = torch.cat([stats.reshape(-1), flag.to(torch.float32)])
            dist.all_reduce(packed, group=mi.group)
            stats, flag = packed[:-1].reshape(stats.shape).contiguous(), (packed[-1:] > 0).to(torch.int32)
        if not (xq and yq) and int(flag.item()) != 0:            # only map operands can be negative
            raise InvalidArgumentError('Condition x >= 0 did not hold element-wise')
        out = torch.empty(items, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib.nrt_mi_finalize_f32(ptr(stats), items, nbx, nby, 1e-7, ptr(out), stream_ptr(dev)))
        ctx.save_for_backward(x, y, cx, cy, mmx, mmy, stats)
        ctx.cfg = (mi, xq, yq, nbx, nby, B, C, nv)
        return out

    @staticmethod
    def backward(ctx, g):
        x, y, cx, cy, mmx, mmy, stats = ctx.saved_tensors
        mi, xq, yq, nbx, nby, B, C, nv = ctx.cfg
        dev = x.device
        items = B * C
        g = g.contiguous().to(torch.float32)
        gstats = torch.empty_like(stats)
        gx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        gy = torch.empty_like(y) if ctx.needs_input_grad[1] else None
        if gx is None and gy is None:
            return (None,) * 10
        # the centres move with the data only when they come from the tensor's min / max
        need_dc = (xq and mmx is not None and gx is not None) or (yq and mmy is not None and gy is not None)
        dcen = torch.zeros((2, 34), dtype=torch.float32, device=dev) if need_dc else None
        wsb = lib.nrt_mi_bwd_workspace_bytes(items) if need_dc else 0
        ws = _workspace(dev, wsb) if need_dc else None
        with torch.cuda.device(dev):
            check(lib.nrt_mi_finalize_bwd_f32(ptr(stats), ptr(g), items, nbx, nby, 1e-7, ptr(gstats), stream_ptr(dev)))
            check(lib.nrt_mi_bwd_f32(ptr(x), nv * x.shape[-1], x.shape[-1], int(xq), nbx, ptr(cx),
                                     ptr(y), nv * y.shape[-1], y.shape[-1], int(yq), nby, ptr(cy),
                                     B, C, nv, float(mi.soft_bin_alpha), float(mi.min_clip), float(mi.max_clip),
                                     ptr(gstats), ptr(gx), ptr(gy), ptr(dcen), ptr(ws), wsb, stream_ptr(dev)))
            if need_dc:
                if mi.group is not None:
                    import torch.distributed as dist
                    dist.all_reduce(dcen, group=mi.group)
                if xq and mmx is not None and gx is not None:
                    check(lib.nrt_mi_minmax_bwd_f32(ptr(x), x.numel(), ptr(mmx), ptr(dcen[0]), nbx, ptr(gx), stream_ptr(dev)))
                if yq and mmy is not None and gy is not None:
                    check(lib.nrt_mi_minmax_bwd_f32(ptr(y), y.numel(), ptr(mmy), ptr(dcen[1]), nby, ptr(gy), stream_ptr(dev)))
        return (gx, gy) + (None,) * 8


# ---------------------------------------------------------------------------------------
# MutualInformation (reference metrics.py:41-336)
# ---------------------------------------------------------------------------------------
class MutualInformation:
    """
    Soft mutual information between volumes, segmentations, or a volume and a segmentation
    (reference metrics.py:41-336): `volumes`, `segs`, `volume_seg`, `channelwise`, `maps`.

    The soft quantisation (neurite.utils.soft_quantize) is fused into the joint-histogram kernel
    (nrt_mi_hist_f32): a volume pair is read once and the [nb, V] x [V, nb] contraction runs on the
    tensor cores.  Differences from the reference, both where the reference cannot run at all:
    explicit `bin_centers` work here (the reference's `_soft_sim_map` passes both `bin_centers` and
    `nb_bins` to soft_quantize, which asserts -- metrics.py:329-331 vs utils.py:1141-1143), and the
    constructor does not print alpha (metrics.py:114).  Differentiable (nrt_mi_bwd_f32), including the
    path through the data-dependent bin centres (min / max of the tensor), like TF autodiff.

    `group`: torch.distributed group over which every item's voxel range is sharded; the bin range
    (min/max) and the [nb*nb + 2 nb] sums are all-reduced before the finalise kernel.
    """

    def __init__(self, bin_centers=None, nb_bins=None, soft_bin_alpha=None, min_clip=None, max_clip=None,
                 group=None):
        self.bin_centers = None
        if bin_centers is not None:
            self.bin_centers = np.asarray(bin_centers, dtype=np.float32)
            assert nb_bins is None, 'cannot provide both bin_centers and nb_bins'
            nb_bins = self.bin_centers.shape[0]
        self.nb_bins = nb_bins
        if bin_centers is None and nb_bins is None:
            self.nb_bins = 16
        self.min_clip = -np.inf if min_clip is None else min_clip
        self.max_clip = np.inf if max_clip is None else max_clip
        self.soft_bin_alpha = soft_bin_alpha
        if self.soft_bin_alpha is None:
            # metrics.py:105-113, fp32 like tf.square / the tensor division
            f32 = np.float32
            if self.bin_centers is None:
                sigma = f32(0.5 / (self.nb_bins - 1))
            else:
                sigma = f32(0.5) * f32(np.mean(np.diff(self.bin_centers), dtype=np.float64))
            self.soft_bin_alpha = f32(1) / (f32(2) * (sigma * sigma))
        self.group = group

    # -- helpers ---------------------------------------------------------------------------
    def _range(self, x32):
        """device [min, max] of the whole tensor (over every rank's shard with `group`), or None
        when the bin centres are explicit."""
        from . import utils
        return None if self.bin_centers is not None else utils.minmax(x32, self.group)

    def _centers(self, x32, mm=None):
        from . import utils
        if self.bin_centers is not None:
            return torch.as_tensor(self.bin_centers, device=x32.device)
        return utils.bin_centers_from_range(self._range(x32) if mm is None else mm, self.nb_bins)

    def _hist(self, x, xq, nbx, y, yq, nby, B, C, nv):
        """x, y: contiguous fp32 [B, nv, stride]; *q = soft-quantise that operand."""
        return _MiFn.apply(x, y, self, bool(xq), bool(yq), int(nbx), int(nby), int(B), int(C), int(nv))

    @staticmethod
    def _bvc(t):
        t = t.to(torch.float32)
        return t.reshape(t.shape[0], -1, t.shape[-1]).contiguous()

    # -- reference API -----------------------------------------------------------------------
    def volumes(self, x, y):
        """MI per batch item of two single-channel volumes [bs, ..., 1] -> [bs] (metrics.py:116-138)."""
        if x.shape[-1] != 1 or y.shape[-1] != 1:
            raise InvalidArgumentError('volume_mi requires two single-channel volumes. See channelwise().')
        return self.channelwise(x, y).reshape(-1)

    def segs(self, x, y):
        """MI of two probabilistic segmentations [bs, ..., nb_labels] -> [bs] (metrics.py:140-152)."""
        return self.maps(x, y)

    def volume_seg(self, x, y):
        """MI of a volume [bs, ..., 1] and a probabilistic segmentation (either order) (metrics.py:154-183)."""
        require_cuda(x, y)
        cxn, cyn = x.shape[-1], y.shape[-1]
        if min(cxn, cyn) != 1:
            raise InvalidArgumentError('volume_seg_mi requires one single-channel volume.')
        if not max(cxn, cyn) > 1:
            raise InvalidArgumentError('volume_seg_mi requires one multi-channel segmentation.')
        vol, seg = (x, y) if cxn == 1 else (y, x)          # MI is symmetric in its arguments
        nb = int(self.nb_bins)
        if tuple(vol.shape[:-1]) + (nb,) != tuple(seg.shape):
            raise InvalidArgumentError('shapes %s and %s differ' % (tuple(vol.shape[:-1]) + (nb,), tuple(seg.shape)))
        v, s = self._bvc(vol), self._bvc(seg)
        return self._hist(v, True, nb, s, False, s.shape[-1], v.shape[0], 1, v.shape[1])

    def channelwise(self, x, y):
        """MI(x[..., i], y[..., i]) for every batch item and channel: [bs, ..., C] -> [bs, C]
        (metrics.py:185-225); bins span the min/max of the whole tensor, as in the reference."""
        require_cuda(x, y)
        if tuple(x.shape) != tuple(y.shape):
            raise InvalidArgumentError('volume shapes do not match')
        xv, yv = self._bvc(x), self._bvc(y)
        B, nv, C = xv.shape
        nb = int(self.nb_bins)
        mi = self._hist(xv, True, nb, yv, True, nb, B, C, nv)
        return mi.reshape(B, C)

    def maps(self, x, y):
        """MI per batch item of two probability / similarity maps [bs, ..., B] -> [bs] (metrics.py:227-292)."""
        require_cuda(x, y)
        if tuple(x.shape) != tuple(y.shape):
            raise InvalidArgumentError('shapes %s and %s differ' % (tuple(x.shape), tuple(y.shape)))
        xv, yv = self._bvc(x), self._bvc(y)
        B, nv, nb = xv.shape
        return self._hist(xv, False, nb, yv, False, nb, B, 1, nv)

    def _soft_log_sim_map(self, x):
        from . import utils
        return utils.soft_quantize(x, alpha=self.soft_bin_alpha, bin_centers=self.bin_centers,
                                   nb_bins=None if self.bin_centers is not None else self.nb_bins,
                                   min_clip=self.min_clip, max_clip=self.max_clip, return_log=True)

    def _soft_sim_map(self, x):
        from . import utils
        return utils.soft_quantize(x, alpha=self.soft_bin_alpha, bin_centers=self.bin_centers,
                                   nb_bins=None if self.bin_centers is not None else self.nb_bins,
                                   min_clip=self.min_clip, max_clip=self.max_clip, return_log=False)
