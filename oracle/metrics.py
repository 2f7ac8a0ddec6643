"""
numpy fp32 restatement of Dice and the label-weighted categorical cross-entropy.
TEST INFRASTRUCTURE (see oracle/__init__.py).

Follows adalca/neurite: neurite/tf:
    metrics.py:352-413   Dice.__init__ (argument checks)
    metrics.py:415-482   Dice.dice
    metrics.py:484-510   Dice.mean_dice
    utils/utils.py:1175-1226  batch_channel_flatten / flatten_axes
    losses.py:68-95      loss = -dice, mean_loss = -mean_dice
    metrics.py:619-650   CategoricalCrossentropy (label weights) + the Keras formula
                         (third party, TF unpinned): p/=sum p; clip(p, 1e-7, 1-1e-7);
                         -sum t log p; mean over all B*V elements.

Reductions use float64 accumulation and round once to fp32: TF's reduction order is
unspecified, so the GPU kernels are compared against the correctly-rounded sum with the
1e-5 relative tolerance north_star states.
"""
import warnings

import numpy as np

F32 = np.float32


class RangeError(ValueError):
    """Stands in for tf.errors.InvalidArgumentError raised by tf.debugging asserts."""


def flatten_axes(x, axes):
    """utils.py:1195-1226."""
    assert isinstance(axes, (list, tuple, range)), 'axes must be list or tuple of axes to be flattened'
    assert np.all(np.diff(axes) == 1), 'axes need to be contiguous'
    if axes[0] < 0:
        assert axes[-1] < 0, 'if one axis is negative, all have to be negative'
    assert axes[-1] < x.ndim, 'axis %d outside max axis %d' % (axes[-1], x.ndim - 1)
    shp = list(x.shape)
    new = shp[:axes[0]] + [-1]
    if axes[-1] < x.ndim - 1 and not (axes[-1] == -1):
        new += shp[axes[-1] + 1:]
    return np.reshape(x, new)


def batch_channel_flatten(x):
    """utils.py:1175-1188."""
    return flatten_axes(x, range(1, x.ndim - 1))


def _divide_no_nan(a, b):
    out = np.zeros(np.broadcast(a, b).shape, dtype=np.result_type(a, b))
    np.divide(a, b, out=out, where=(b != 0))
    return out


def _sum_f32(x, axis, keepdims=False):
    return np.sum(x, axis=axis, dtype=np.float64, keepdims=keepdims).astype(F32)


def _one_hot(idx, depth):
    idx = np.asarray(idx)
    out = np.zeros(idx.shape + (depth,), dtype=F32)
    valid = (idx >= 0) & (idx < depth)
    np.put_along_axis(out, np.where(valid, idx, 0)[..., None].astype(np.int64),
                      valid[..., None].astype(F32), axis=-1)
    return out


class Dice:
    """metrics.py:339-519 (+ losses.py:46-95)."""

    def __init__(self, dice_type='soft', input_type='prob', nb_labels=None, weights=None,
                 check_input_limits=True, laplace_smoothing=0., normalize=False):
        self.dice_type = dice_type
        self.input_type = input_type
        self.nb_labels = nb_labels
        self.weights = weights
        self.normalize = normalize
        self.check_input_limits = check_input_limits
        self.laplace_smoothing = laplace_smoothing
        assert self.input_type in ['prob', 'max_label']                   # :406
        if self.dice_type == 'hard' and self.input_type == 'max_label':
            assert self.nb_labels is not None, 'If doing hard Dice need nb_labels'   # :408-409
        if self.dice_type == 'soft':
            assert self.input_type in ['prob', 'one_hot'], \
                'if doing soft Dice, must use probabilistic (one_hot)encoding'       # :411-413

    def dice(self, y_true, y_pred):
        y_true = np.asarray(y_true)
        y_pred = np.asarray(y_pred)
        if self.input_type in ['prob', 'one_hot']:
            y_true = y_true.astype(F32)
            y_pred = y_pred.astype(F32)
            if self.normalize:                                            # :434-436
                y_true = _divide_no_nan(y_true, _sum_f32(y_true, -1, keepdims=True))
                y_pred = _divide_no_nan(y_pred, _sum_f32(y_pred, -1, keepdims=True))
            if self.check_input_limits:                                   # :439-444
                msg = 'value outside range'
                for y in (y_true, y_pred):
                    if not np.all(y >= 0.):
                        raise RangeError(msg)
                for y in (y_true, y_pred):
                    if not np.all(y <= 1.):
                        raise RangeError(msg)
        if self.dice_type == 'hard':                                      # :450-468
            if self.input_type == 'prob':
                warnings.warn('You are using ne.metrics.Dice with probabilistic inputs'
                              'and computing *hard* dice.')
                if self.nb_labels is None:
                    self.nb_labels = y_pred.shape[-1]
                y_pred = np.argmax(y_pred, axis=-1)
                y_true = np.argmax(y_true, axis=-1)
            y_pred = _one_hot(np.asarray(y_pred).astype(np.int64), self.nb_labels)
            y_true = _one_hot(np.asarray(y_true).astype(np.int64), self.nb_labels)
        y_true = batch_channel_flatten(y_true)                            # :471-472
        y_pred = batch_channel_flatten(y_pred)
        top = F32(2) * _sum_f32(y_true * y_pred, 1)                       # :476
        bottom = _sum_f32(np.square(y_true), 1) + _sum_f32(np.square(y_pred), 1)   # :477
        if self.laplace_smoothing > 0:                                    # :478-482
            eps = F32(self.laplace_smoothing)
            return (top + eps) / (bottom + eps)
        return _divide_no_nan(top, bottom)

    def mean_dice(self, y_true, y_pred):
        dice_metric = self.dice(y_true, y_pred)                           # :499
        if self.weights is not None:                                      # :502-505
            w = np.asarray(self.weights)
            assert len(w.shape) == 2, \
                'weights should be a matrix broadcastable to [batch_size, nb_labels]'
            dice_metric = dice_metric * w.astype(F32)
        m = F32(np.mean(dice_metric, dtype=np.float64))                   # :508
        if not np.isfinite(m):
            raise RangeError('metric not finite')                         # :509
        return m

    def loss(self, y_true, y_pred):                                       # losses.py:68-80
        return -self.dice(y_true, y_pred)

    def mean_loss(self, y_true, y_pred):                                  # losses.py:82-95
        return -self.mean_dice(y_true, y_pred)


def categorical_crossentropy(y_true, y_pred, label_weights=None, sample_weight=None,
                             from_logits=False, label_smoothing=0., reduction='sum_over_batch_size',
                             per_element=False):
    """metrics.py:640-650, then Keras CategoricalCrossentropy.__call__ (axis=-1).

    Returns the reduced scalar (fp32), or the per-element loss [B,*S] if per_element /
    reduction == 'none'."""
    y_true = np.asarray(y_true, dtype=F32)
    y_pred = np.asarray(y_pred, dtype=F32)
    if label_weights is not None:
        lw = np.asarray(label_weights)
        if lw.shape[-1] != y_pred.shape[-1]:
            raise ValueError(f'Label weights must be of len {y_pred.shape[-1]}, but got {lw.shape[-1]}.')
        y_true = lw.astype(F32) * y_true                                  # :648
    C = y_pred.shape[-1]
    if label_smoothing:
        ls = F32(label_smoothing)
        y_true = y_true * (F32(1) - ls) + ls / F32(C)
    if from_logits:
        m = np.max(y_pred, axis=-1, keepdims=True)
        z = y_pred - m
        lse = np.log(np.sum(np.exp(z.astype(np.float64)), axis=-1, keepdims=True))
        logp = z.astype(np.float64) - lse
    else:
        p = y_pred / _sum_f32(y_pred, -1, keepdims=True)
        eps = F32(1e-7)
        p = np.clip(p, eps, F32(1) - eps)
        logp = np.log(p.astype(np.float64))
    loss = (-np.sum(y_true.astype(np.float64) * logp, axis=-1)).astype(F32)      # [B,*S]
    if sample_weight is not None:
        loss = loss * np.asarray(sample_weight, dtype=F32)
    if per_element or reduction == 'none':
        return loss
    if reduction == 'sum':
        return F32(np.sum(loss, dtype=np.float64))
    return F32(np.sum(loss, dtype=np.float64) / loss.size)
