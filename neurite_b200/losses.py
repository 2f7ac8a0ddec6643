"""
neurite_b200.losses -- the loss shells of neurite.losses (adalca/neurite: neurite/tf/losses.py:46-205):
`loss = -dice` ([batch, nb_labels]), `mean_loss = -mean_dice` (scalar), and
CategoricalCrossentropy.loss = cce.  Bound methods are `(y_true, y_pred) -> Tensor` callables,
the protocol the reference hands to model.compile(loss=...) and callbacks.PredictMetrics.
"""
from . import metrics
from .metrics import MutualInformation  # noqa: F401  (reference losses.py:40-43 re-exports it)


class _DiceLossMixin:
    def loss(self, y_true, y_pred):
        """dice loss (negative Dice score), [batch_size, nb_labels] -- losses.py:68-80."""
        return -self.dice(y_true, y_pred)

    def mean_loss(self, y_true, y_pred):
        """negative mean dice, optionally weighted -- losses.py:82-95."""
        return -self.mean_dice(y_true, y_pred)


class Dice(_DiceLossMixin, metrics.Dice):
    """losses.py:46-95."""


class SoftDice(_DiceLossMixin, metrics.SoftDice):
    """losses.py:98-143."""


class HardDice(_DiceLossMixin, metrics.HardDice):
    """losses.py:146-190."""


class CategoricalCrossentropy(metrics.CategoricalCrossentropy):
    """losses.py:193-205."""

    def loss(self, *args, **kwargs):
        return self.cce(*args, **kwargs)
