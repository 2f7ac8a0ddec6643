"""
neurite_b200 -- H100-native (sm_90a) implementation of neurite's per-volume hot path:
interpn / resize / SpatialTransformer, LocallyConnected3D, Dice and the label-weighted
categorical cross-entropy, behind neurite's own call signatures.

    import neurite_b200 as ne
    ne.utils.interpn(vol, loc)            ne.layers.Resize(2)(x)
    ne.layers.SpatialTransformer()([vol, flow])
    ne.layers.LocallyConnected3D(16, 3)(x)
    ne.losses.Dice().loss(y_true, y_pred) ne.losses.CategoricalCrossentropy(label_weights=w).loss(t, p)

Tensors are torch CUDA tensors, channels-last ([batch, *spatial, channels]) like the
reference.  All arithmetic runs in hand-written CUDA behind a C ABI
(include/neurite_b200.h, neurite_b200/lib/libneurite_b200.so); importing the package
fails if that library has not been built -- there is no CPU fallback.
"""
__version__ = '0.1'

from . import _lib  # noqa: F401  (raises ImportError when the CUDA library is missing)
from . import utils, layers, metrics, losses, dist, models, augment  # noqa: F401
from .utils import interpn, resize, zoom, transform  # noqa: F401
