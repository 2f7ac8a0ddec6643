"""
oracle/ -- CPU restatement of the reference's hot path.  TEST INFRASTRUCTURE ONLY.

This package is the *checker*, never the product.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it.  ``neurite_b200`` (the product) never imports, links or calls it.

What it restates (all citations are into adalca/neurite @ 7c4b05e):

  interp.py   neurite/tf/utils/utils.py:73-220   interpn (linear / nearest / fill_value)
              neurite/tf/utils/utils.py:223-265  resize / zoom
              neurite/tf/utils/utils.py:333-476  ndgrid / meshgrid / volshape_to_*
              neurite/tf/utils/utils.py:1068-1092 sub2ind2d / prod_n
              voxelmorph SpatialTransformer (third party, contract in SURVEY.md 8c)
  lc3d.py     neurite/tf/layers.py:951-1047, 1098-1101, 1126-1197  LocallyConnected3D impl 1
  metrics.py  neurite/tf/metrics.py:415-510      Dice.dice / mean_dice
              neurite/tf/utils/utils.py:1175-1226 batch_channel_flatten / flatten_axes
              neurite/tf/metrics.py:640-650 + Keras CategoricalCrossentropy formula
  mi.py       neurite/tf/metrics.py:41-336       MutualInformation (volumes / segs / volume_seg /
              channelwise / maps), neurite/tf/utils/utils.py:1099-1172 soft_quantize;
              plus a float64 torch restatement of the same graph as the GRADIENT oracle
  grad.py     differentiable torch restatements of interpn / warp / resize / VecInt / Dice / CCE /
              LocallyConnected3D (the GRADIENT oracle of the other ops) and the per-element
              gradient error bound the GPU gradient tests use
  forward.py  float64 forward references (Dice with normalize, hard-Dice counts, separable
              convolution, MI joint histograms and bin centres) and the per-element bound of each
              forward kernel, its depth derived from the launch geometry
  conv.py     neurite/tf/utils/utils.py:581-751  gaussian_kernel / separable_conv,
              neurite/tf/layers.py:251-364 GaussianBlur, utils.py:754-826 subsample_axis
  c/          the same arithmetic as fused C99 + OpenMP loops (fast enough for full-size
              160x192x224 parity and for the multi-threaded CPU baseline)

Pinning status
--------------
The reference ships no tests, fixtures or golden vectors for this path (SURVEY.md 0.2),
and TensorFlow cannot be imported in this image.  Parity is pinned as follows:

  * tests/golden/*.npz were produced by executing the REFERENCE'S OWN python source
    (imported from a reference checkout, unmodified) on top of ``tools/tfshim`` -- a numpy
    implementation of the ~60 TensorFlow/Keras ops those functions call.  The generating
    script is tools/gen_golden.py.  The algorithm (clip/cast order, corner order,
    weight products, fill mask, Dice sums, patch ordering) is therefore the
    reference's, op for op; only the leaf ops (floor, clip, gather, ...) are numpy's.
  * the docstring known answers the reference does contain (SURVEY.md 4) are asserted
    in tests/test_oracle.py.
  * independent cross-checks: scipy.ndimage.map_coordinates(order=1, mode='nearest'),
    torch grid_sample(border, align_corners=True), F.conv3d with position-shared weights,
    scipy.ndimage.correlate1d and F.conv3d for the separable convolutions, the plug-in
    entropy / hard-histogram limits for MutualInformation.
  * third-party arithmetic that is NOT in the reference (voxelmorph
    SpatialTransformer, Keras CategoricalCrossentropy, tf.linspace, tf.nn.convolution) is
    restated from its published definition: for those pieces parity is UNPINNED by the
    reference repo itself and says so in DESIGN.md.
"""
from . import conv, interp, lc3d, metrics, mi  # noqa: F401
