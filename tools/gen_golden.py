#!/usr/bin/env python
"""
tools/gen_golden.py -- generate tests/golden/*.npz by EXECUTING THE REFERENCE'S OWN SOURCE.

    python tools/gen_golden.py REFERENCE_ROOT     # a checkout of adalca/neurite @ 7c4b05e

The reference (adalca/neurite @ 7c4b05e) is pure Python on TensorFlow, and TensorFlow is
not installable here.  tools/tfshim.py supplies a numpy implementation of the leaf TF ops;
this script imports `neurite` from REFERENCE_ROOT unmodified and calls

    neurite.utils.interpn / resize / volshape_to_meshgrid           (tf/utils/utils.py)
    neurite.layers.Resize, neurite.layers.LocallyConnected3D         (tf/layers.py)
    neurite.metrics.Dice / SoftDice / HardDice, neurite.losses.*     (tf/metrics.py, losses.py)
    neurite.metrics.CategoricalCrossentropy                          (label-weight wrapper)

on seeded inputs, storing inputs + outputs.  Each fixture's `provenance` field says which
reference symbol produced it.  Two fixtures are *compositions by contract* because their
arithmetic lives in packages absent from the reference (SURVEY.md 8c): `st_*`
(voxelmorph SpatialTransformer = reference meshgrid + flow -> reference interpn) and the
Keras CCE formula inside tfshim.  They are labelled provenance='contract'.

The fixtures are committed: tests never read the reference at run time.
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import tfshim  # noqa: E402

if len(sys.argv) < 2:
    raise SystemExit('usage: python tools/gen_golden.py REFERENCE_ROOT [GROUP ...]')
ne = tfshim.install(sys.argv[1])
T = tfshim.Tensor
OUT = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
os.makedirs(OUT, exist_ok=True)
F32 = np.float32


def npy(x):
    return np.asarray(x.numpy() if isinstance(x, T) else x)


def save(name, provenance, **arrays):
    arrays['provenance'] = np.array(provenance)
    path = os.path.join(OUT, name + '.npz')
    np.savez_compressed(path, **arrays)
    print('%-34s %8.1f KB  %s' % (name, os.path.getsize(path) / 1024, provenance))


def identity_plus(shape, rng, amp):
    grid = np.stack(np.meshgrid(*[np.arange(s, dtype=F32) for s in shape], indexing='ij'), -1)
    return (grid + rng.uniform(-amp, amp, grid.shape).astype(F32)).astype(F32)


# ---------------------------------------------------------------------------------------
# interpn
# ---------------------------------------------------------------------------------------
def gen_interpn():
    ref = 'reference neurite/tf/utils/utils.py:73-220 interpn on tfshim'
    # cfg1 of BASELINE.json: 32^3, linear, seed 0/1 (SURVEY.md 8d)
    vol = np.random.default_rng(0).standard_normal((32, 32, 32)).astype(F32)
    loc = identity_plus((32, 32, 32), np.random.default_rng(1), 3.0)
    out = npy(ne.utils.interpn(T(vol), T(loc)))
    save('interpn_cfg1_linear_32', ref, vol=vol, loc=loc, out=out, method=np.array('linear'))

    rng = np.random.default_rng(10)
    shape = (9, 11, 13)
    for C in (None, 1, 3, 4, 5):
        vshape = shape if C is None else shape + (C,)
        vol = rng.standard_normal(vshape).astype(F32)
        loc = identity_plus(shape, rng, 4.0)                       # plenty out of range
        # exact integers, exact .5 ties, exact edges
        loc[0, 0, :5] = [[0, 0, 0], [8, 10, 12], [0.5, 1.5, 2.5], [-0.0, 10.0, 12.0], [8.0, 0, 3.5]]
        loc[1, 0, :3] = [[-1e-7, 3, 3], [8.0000001, 3, 3], [3, 10.000001, 3]]
        tag = 'c%s' % ('none' if C is None else C)
        for method in ('linear', 'nearest'):
            for fill in (None, 0.0, -7.25):
                out = npy(ne.utils.interpn(T(vol), T(loc), interp_method=method, fill_value=fill))
                save('interpn_3d_%s_%s_fill%s' % (tag, method, 'none' if fill is None else str(fill).replace('.', 'p').replace('-', 'm')),
                     ref, vol=vol, loc=loc, out=out, method=np.array(method),
                     fill=np.array(np.nan if fill is None else fill, dtype=F32))

    # loc grid of a different size than the volume, loc as list, 2-D and 1-D
    vol = rng.standard_normal((7, 10, 2)).astype(F32)
    loc = rng.uniform(-2, 11, (5, 6, 2)).astype(F32)
    for method in ('linear', 'nearest'):
        out = npy(ne.utils.interpn(T(vol), [T(loc[..., 0]), T(loc[..., 1])], interp_method=method))
        save('interpn_2d_list_%s' % method, ref, vol=vol, loc=loc, out=out, method=np.array(method),
             fill=np.array(np.nan, dtype=F32))
    vol = rng.standard_normal((17,)).astype(F32)
    loc = rng.uniform(-3, 20, (23, 1)).astype(F32)
    loc[:4, 0] = [.5, 1.5, 2.5, 3.5]
    for method in ('linear', 'nearest'):
        out = npy(ne.utils.interpn(T(vol), T(loc), interp_method=method, fill_value=1.5))
        save('interpn_1d_%s' % method, ref, vol=vol, loc=loc, out=out, method=np.array(method),
             fill=np.array(1.5, dtype=F32))
    # more than three dimensions: the reference's interpn is N-D (utils.py:106-120, 2^D corners in product order)
    for D, vshape, C in ((4, (5, 6, 4, 7), 2), (5, (3, 4, 3, 5, 4), None)):
        vol = rng.standard_normal(vshape if C is None else vshape + (C,)).astype(F32)
        loc = np.stack([rng.uniform(-1.5, s + 0.5, (6, 7)) for s in vshape], -1).astype(F32)
        loc[0, 0] = 0
        loc[0, 1] = [s - 1 for s in vshape]
        loc[0, 2] = [0.5 + (d % 2) for d in range(D)]
        for method, fill in (('linear', None), ('linear', 2.5), ('nearest', 0.0)):
            out = npy(ne.utils.interpn(T(vol), T(loc), interp_method=method, fill_value=fill))
            save('interpn_%dd_%s_fill%s' % (D, method, 'none' if fill is None else str(fill).replace('.', 'p')), ref,
                 vol=vol, loc=loc, out=out, method=np.array(method), fill=np.array(np.nan if fill is None else fill, dtype=F32))
    # integer-valued label volume + nearest + fill 0: the only in-repo usage (models.py:806-809)
    vol = rng.integers(0, 16, (8, 9, 10, 1)).astype(F32)
    loc = identity_plus((8, 9, 10), rng, 2.5)
    out = npy(ne.utils.interpn(T(vol), T(loc), interp_method='nearest', fill_value=0))
    save('interpn_labels_nearest_fill0', ref, vol=vol, loc=loc, out=out, method=np.array('nearest'),
         fill=np.array(0, dtype=F32))


# ---------------------------------------------------------------------------------------
# resize / Resize layer
# ---------------------------------------------------------------------------------------
def gen_resize():
    ref = 'reference neurite/tf/utils/utils.py:223-265 resize on tfshim (tf.linspace restated)'
    rng = np.random.default_rng(20)
    cases = [((6, 7, 8, 2), 2), ((6, 7, 8, 1), 1.5), ((9, 8, 7, 3), 0.7), ((5, 6, 4, 2), [2, 1, 3]),
             ((8, 9, 2), 2.5), ((12, 1), 3)]
    for i, (shape, z) in enumerate(cases):
        vol = rng.standard_normal(shape).astype(F32)
        for method in ('linear', 'nearest'):
            out = npy(ne.utils.resize(T(vol), z, interp_method=method))
            save('resize_%d_%s' % (i, method), ref, vol=vol, zoom=np.asarray(z, dtype=np.float64),
                 out=out, method=np.array(method))
    x = rng.standard_normal((2, 6, 5, 4, 3)).astype(F32)
    lay = ne.layers.Resize(2)
    out = npy(lay(T(x)))
    save('resize_layer_zoom2', 'reference neurite/tf/layers.py:91-185 Resize.call on tfshim',
         x=x, zoom=np.asarray(2.0), out=out, method=np.array('linear'))
    lay = ne.layers.Resize([0.5, 1.5, 2], interp_method='nearest')
    out = npy(lay(T(x)))
    save('resize_layer_list_nearest', 'reference neurite/tf/layers.py:91-185 Resize.call on tfshim',
         x=x, zoom=np.asarray([0.5, 1.5, 2]), out=out, method=np.array('nearest'))


# ---------------------------------------------------------------------------------------
# SpatialTransformer (contract composition; voxelmorph absent)
# ---------------------------------------------------------------------------------------
def gen_spatial_transformer():
    prov = ('contract: voxelmorph SpatialTransformer (absent) = reference volshape_to_meshgrid '
            '(utils.py:356-379, ij) + flow -> reference interpn (utils.py:73-220) on tfshim')
    rng = np.random.default_rng(30)
    for name, shape, C, method, fill, amp in [
            ('st_3d_c1_linear', (10, 12, 16), 1, 'linear', None, 3.0),
            ('st_3d_c1_linear_fill', (10, 12, 16), 1, 'linear', 0.0, 3.0),
            ('st_3d_c1_big', (10, 12, 16), 1, 'linear', None, 9.0),
            ('st_3d_c4_linear', (6, 8, 12), 4, 'linear', None, 2.0),
            ('st_3d_c16_linear', (5, 6, 8), 16, 'linear', None, 2.0),
            ('st_3d_c3_linear', (5, 6, 8), 3, 'linear', None, 2.0),
            ('st_3d_labels_nearest_fill0', (8, 8, 12), 1, 'nearest', 0.0, 3.0),
            ('st_2d_c2_linear', (9, 12), 2, 'linear', None, 2.5)]:
        B = 2
        nd = len(shape)
        vol = rng.standard_normal((B,) + shape + (C,)).astype(F32)
        if 'labels' in name:
            vol = rng.integers(0, 16, vol.shape).astype(F32)
        flow = rng.uniform(-amp, amp, (B,) + shape + (nd,)).astype(F32)
        outs = []
        for b in range(B):
            mesh = ne.utils.volshape_to_meshgrid(shape, indexing='ij')
            tf = sys.modules['tensorflow']
            loc = [tf.cast(mesh[d], 'float32') + T(flow[b, ..., d]) for d in range(nd)]
            outs.append(npy(ne.utils.interpn(T(vol[b]), loc, interp_method=method, fill_value=fill)))
        save(name, prov, vol=vol, flow=flow, out=np.stack(outs, 0), method=np.array(method),
             fill=np.array(np.nan if fill is None else fill, dtype=F32))


# ---------------------------------------------------------------------------------------
# Dice / CCE
# ---------------------------------------------------------------------------------------
def gen_dice():
    ref = 'reference neurite/tf/metrics.py:339-616 + losses.py:46-190 on tfshim'
    rng = np.random.default_rng(40)
    B, S, L = 3, (6, 7, 8), 16
    labels = rng.integers(0, L, (B,) + S)
    y_true = np.eye(L, dtype=F32)[labels]
    logits = rng.standard_normal((B,) + S + (L,)).astype(F32)
    e = np.exp(logits - logits.max(-1, keepdims=True))
    y_pred = (e / e.sum(-1, keepdims=True)).astype(F32)
    y_pred = np.clip(y_pred, 0, 1)
    lab_pred = rng.integers(0, L, (B,) + S)
    w = rng.uniform(0.5, 2, (1, L)).astype(F32)

    d = ne.losses.Dice()
    save('dice_soft_default', ref, y_true=y_true, y_pred=y_pred,
         dice=npy(d.dice(T(y_true), T(y_pred))), loss=npy(d.loss(T(y_true), T(y_pred))),
         mean_dice=npy(d.mean_dice(T(y_true), T(y_pred))), mean_loss=npy(d.mean_loss(T(y_true), T(y_pred))))
    d = ne.losses.SoftDice(weights=T(w), laplace_smoothing=0.1)
    save('dice_soft_laplace_weights', ref, y_true=y_true, y_pred=y_pred, weights=w,
         dice=npy(d.dice(T(y_true), T(y_pred))), mean_loss=npy(d.mean_loss(T(y_true), T(y_pred))))
    d = ne.losses.Dice(normalize=True)
    un_t = (y_true * rng.uniform(0.2, 1.0, y_true.shape[:-1] + (1,))).astype(F32)
    un_p = (y_pred * rng.uniform(0.2, 1.0, y_pred.shape[:-1] + (1,))).astype(F32)
    un_t[0, 0, 0, 0] = 0       # an all-zero voxel: divide_no_nan -> 0
    save('dice_soft_normalize', ref, y_true=un_t, y_pred=un_p, dice=npy(d.dice(T(un_t), T(un_p))))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        d = ne.losses.Dice(dice_type='hard', input_type='prob')
        save('dice_hard_prob', ref, y_true=y_true, y_pred=y_pred, dice=npy(d.dice(T(y_true), T(y_pred))))
    d = ne.losses.HardDice(L)
    save('dice_hard_max_label', ref, y_true=labels.astype(np.int32), y_pred=lab_pred.astype(np.int32),
         nb_labels=np.array(L), dice=npy(d.dice(T(labels.astype(np.int32)), T(lab_pred.astype(np.int32)))),
         mean_loss=npy(d.mean_loss(T(labels.astype(np.int32)), T(lab_pred.astype(np.int32)))))
    # disjoint / absent labels -> 0/0 -> 0 ; 5 labels (not a multiple of 4); 2-D volumes
    L2 = 5
    lab = rng.integers(0, 3, (2, 9, 10))
    t = np.eye(L2, dtype=F32)[lab]
    p = np.eye(L2, dtype=F32)[(lab + 1) % 3]
    d = ne.losses.Dice()
    save('dice_soft_disjoint_L5', ref, y_true=t, y_pred=p, dice=npy(d.dice(T(t), T(p))))
    # range violation
    bad = y_pred.copy()
    bad[1, 2, 3, 4, 5] = 1.5
    try:
        ne.losses.Dice().dice(T(y_true), T(bad))
        raised = ''
    except Exception as ex:                                       # noqa: BLE001
        raised = '%s: %s' % (type(ex).__name__, ex)
    save('dice_range_error', ref, y_true=y_true, y_pred=bad, raised=np.array(raised))

    prov = ('contract: reference label-weight wrapper neurite/tf/metrics.py:640-650 executed on tfshim; '
            'the Keras CategoricalCrossentropy arithmetic underneath is restated (third party)')
    lw = rng.uniform(0.1, 3, (L,)).astype(F32)
    c = ne.losses.CategoricalCrossentropy(label_weights=lw)
    save('cce_label_weights', prov, y_true=y_true, y_pred=y_pred, label_weights=lw,
         loss=npy(c.loss(T(y_true), T(y_pred))))
    c = ne.losses.CategoricalCrossentropy()
    save('cce_plain', prov, y_true=y_true, y_pred=y_pred, loss=npy(c(T(y_true), T(y_pred))))
    try:
        ne.losses.CategoricalCrossentropy(label_weights=lw[:5]).loss(T(y_true), T(y_pred))
        raised = ''
    except ValueError as ex:
        raised = 'ValueError: %s' % ex
    save('cce_bad_weights', prov, raised=np.array(raised))


# ---------------------------------------------------------------------------------------
# LocallyConnected3D
# ---------------------------------------------------------------------------------------
def gen_lc3d():
    ref = 'reference neurite/tf/layers.py:811-1197 LocallyConnected3D (impl 1) on tfshim'
    rng = np.random.default_rng(50)
    cases = [
        ('lc3d_k3_s1_cl', (2, 6, 7, 8, 3), 4, (3, 3, 3), (1, 1, 1), 'channels_last', True),
        ('lc3d_k3_s1_16to16', (1, 5, 5, 6, 16), 16, (3, 3, 3), (1, 1, 1), 'channels_last', True),
        ('lc3d_k321_s212_cl', (2, 7, 6, 9, 2), 5, (3, 2, 1), (2, 1, 2), 'channels_last', True),
        ('lc3d_k2_s1_cf', (2, 3, 5, 6, 5), 4, (2, 2, 2), (1, 1, 1), 'channels_first', True),
        ('lc3d_k3_nobias', (3, 5, 5, 5, 2), 3, 3, (1, 1, 1), 'channels_last', False),
    ]
    for name, xshape, filters, ks, st, fmt, use_bias in cases:
        lay = ne.layers.LocallyConnected3D(filters, ks, strides=st, data_format=fmt, use_bias=use_bias)
        lay.build(xshape)
        kshape = lay.kernel_shape
        oshape = (lay.output_row, lay.output_col, lay.output_z)
        kernel = rng.standard_normal(kshape).astype(F32)
        bias = rng.standard_normal(oshape + (filters,)).astype(F32) if use_bias else None
        lay.kernel = T(kernel)
        lay.bias = T(bias) if use_bias else None
        lay.activation = lambda v: v
        x = rng.standard_normal(xshape).astype(F32)
        out = npy(lay.call(T(x)))
        assert tuple(out.shape) == tuple(lay.compute_output_shape(xshape)), (out.shape, lay.compute_output_shape(xshape))
        save(name, ref, x=x, kernel=kernel, bias=np.zeros(0, F32) if bias is None else bias, out=out,
             kernel_size=np.asarray(lay.kernel_size), strides=np.asarray(lay.strides),
             data_format=np.array(fmt), filters=np.array(filters))


def gen_lc3d_impl():
    """Weight orderings of LocallyConnected3D implementations 2 / 3: the reference's own index generator
    (conv_kernel_idxs, layers.py:1346-1434; build() sorts it, :1012-1021) executed on small geometries.  The fixture
    holds the sorted (out_flat, in_flat) pairs -- the order of the implementation-3 weight vector and the support of the
    implementation-2 mask."""
    ref = 'reference neurite/tf/layers.py:1346-1434 LocallyConnected3D.conv_kernel_idxs (sorted as in build(), :1012-1021)'
    cases = [('lc3d_impl_idx_cl', (4, 5, 3), 2, 3, (2, 3, 2), (1, 1, 1), 'channels_last'),
             ('lc3d_impl_idx_cl_s2', (5, 4, 6), 3, 2, (3, 2, 2), (2, 1, 2), 'channels_last'),
             ('lc3d_impl_idx_cf', (3, 4, 4), 2, 2, (2, 2, 3), (1, 2, 1), 'channels_first')]
    for name, ishape, cin, cout, ks, st, fmt in cases:
        idxs = sorted(ne.layers.LocallyConnected3D.conv_kernel_idxs(input_shape=ishape, kernel_shape=ks, strides=st,
                                                                    padding='valid', filters_in=cin, filters_out=cout,
                                                                    data_format=fmt))
        save(name, ref, idxs=np.asarray(idxs, dtype=np.int64), input_shape=np.asarray(ishape), filters_in=np.array(cin),
             filters_out=np.array(cout), kernel_size=np.asarray(ks), strides=np.asarray(st), data_format=np.array(fmt))


# ---------------------------------------------------------------------------------------
# MutualInformation / soft_quantize  (SURVEY.md 8f-3)
# ---------------------------------------------------------------------------------------
def gen_mi():
    import contextlib
    import io
    ref = 'reference neurite/tf/metrics.py:41-336 MutualInformation + utils.py:1099-1172 soft_quantize on tfshim'
    rng = np.random.default_rng(70)
    S = (9, 10, 11)

    def make_mi(**kw):
        with contextlib.redirect_stdout(io.StringIO()):          # the ctor prints alpha (metrics.py:114)
            return ne.metrics.MutualInformation(**kw)

    # soft_quantize as a tensor op
    x = rng.uniform(-0.2, 1.3, (2,) + S).astype(F32)
    for tag, kw in (('default', {}), ('nb8_alpha', dict(nb_bins=8, alpha=3.5)),
                    ('centers_clip', dict(bin_centers=np.linspace(0, 1, 6).astype(F32), nb_bins=None, alpha=20.,
                                          min_clip=0.1, max_clip=0.9)),
                    ('log', dict(nb_bins=5, alpha=2., return_log=True))):
        out = npy(ne.utils.soft_quantize(T(x), **kw))
        save('softq_' + tag, ref, x=x, out=out, kw=np.array(repr(kw)))

    # volumes: correlated pair (y = smooth function of x + noise), independent pair, identical pair
    a = rng.uniform(0, 1, (3,) + S + (1,)).astype(F32)
    b = np.clip(0.6 * a ** 2 + 0.2 + 0.05 * rng.standard_normal(a.shape), 0, 1).astype(F32)
    c = rng.uniform(0, 1, a.shape).astype(F32)
    for nb in (16, 32, 7):
        mi = make_mi(nb_bins=nb)
        save('mi_volumes_nb%d' % nb, ref, x=a, y=b, nb_bins=np.array(nb), alpha=npy(mi.soft_bin_alpha),
             mi=npy(mi.volumes(T(a), T(b))), mi_indep=npy(mi.volumes(T(a), T(c))), mi_self=npy(mi.volumes(T(a), T(a))))
    mi = make_mi(nb_bins=12, soft_bin_alpha=55.0, min_clip=0.05, max_clip=0.95)
    save('mi_volumes_clip_alpha', ref, x=a, y=b, nb_bins=np.array(12), alpha=np.array(55.0, F32),
         min_clip=np.array(0.05, F32), max_clip=np.array(0.95, F32), mi=npy(mi.volumes(T(a), T(b))))

    # channelwise: 3 channels, bins from the min/max of the whole tensor
    xc = rng.uniform(0, 1, (2,) + S + (3,)).astype(F32)
    yc = np.clip(xc[..., ::-1] * 0.7 + 0.1 * rng.standard_normal(xc.shape), 0, 1).astype(F32)
    mi = make_mi()
    save('mi_channelwise_c3', ref, x=xc, y=yc, mi=npy(mi.channelwise(T(xc), T(yc))))

    # segs / maps: softmax probability maps, 16 and 5 labels
    for L in (16, 5):
        lx = rng.standard_normal((2,) + S + (L,)).astype(F32) * 2
        ly = (lx + rng.standard_normal(lx.shape).astype(F32)).astype(F32)
        px = (np.exp(lx) / np.exp(lx).sum(-1, keepdims=True)).astype(F32)
        py = (np.exp(ly) / np.exp(ly).sum(-1, keepdims=True)).astype(F32)
        save('mi_segs_L%d' % L, ref, x=px, y=py, mi=npy(make_mi().segs(T(px), T(py))))
        if L == 16:
            px16 = px

    # volume_seg: volume vs 16-label map (the quantised volume has nb_bins = 16 channels too)
    v = rng.uniform(0, 1, (2,) + S + (1,)).astype(F32)
    mi = make_mi(nb_bins=16)
    save('mi_volume_seg', ref, vol=v, seg=px16, mi_vs=npy(mi.volume_seg(T(v), T(px16))),
         mi_sv=npy(mi.volume_seg(T(px16), T(v))))

    # error behaviour
    errs = {}
    def rec(name, fn):
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                fn()
            errs[name] = ''
        except Exception as ex:                                    # noqa: BLE001
            errs[name] = '%s: %s' % (type(ex).__name__, ex)
    rec('volumes_two_channels', lambda: make_mi().volumes(T(xc), T(yc)))
    rec('maps_shape_mismatch', lambda: make_mi().maps(T(px), T(py[..., :3])))
    rec('volume_seg_bins_ne_labels', lambda: make_mi(nb_bins=16).volume_seg(T(v), T(px)))
    rec('maps_negative', lambda: make_mi().maps(T(px), T(-py)))
    rec('volume_seg_two_volumes', lambda: make_mi().volume_seg(T(v), T(v)))
    rec('both_centers_and_bins', lambda: ne.metrics.MutualInformation(bin_centers=np.linspace(0, 1, 4), nb_bins=4))
    rec('explicit_centers_volumes', lambda: make_mi(bin_centers=np.linspace(0, 1, 8).astype(F32)).volumes(T(a), T(b)))
    save('mi_errors', ref, **{k: np.array(val) for k, val in errs.items()})


# ---------------------------------------------------------------------------------------
# gaussian_kernel / separable_conv / GaussianBlur  (SURVEY.md 8f-4)
# ---------------------------------------------------------------------------------------
def gen_blur():
    ref = ('reference neurite/tf/utils/utils.py:581-751 gaussian_kernel + separable_conv, layers.py:251-364 '
           'GaussianBlur on tfshim (tf.nn.convolution restated: contract)')
    rng = np.random.default_rng(80)
    for tag, sigma in (('s1', 1.0), ('s0p5', 0.5), ('s2p3', 2.3), ('aniso', [1.0, 0.0, 2.0])):
        ks = ne.utils.gaussian_kernel(sigma, separate=True)
        ks = ks if isinstance(ks, list) else [ks]
        save('gausskernel_' + tag, ref, sigma=np.asarray(sigma, F32), n=np.array(len(ks)),
             **{'k%d' % i: npy(k) for i, k in enumerate(ks)})
    k2 = npy(ne.utils.gaussian_kernel([1.0, 1.5]))
    save('gausskernel_2d_full', ref, sigma=np.asarray([1.0, 1.5], F32), k=k2)

    x3 = rng.standard_normal((2, 9, 12, 40, 2)).astype(F32)
    for tag, sigma in (('s1', 1.0), ('aniso', [1.5, 0.0, 0.7]), ('s3', 3.0)):
        out = npy(ne.layers.GaussianBlur(sigma=sigma)(T(x3)))
        save('blur3d_' + tag, ref, x=x3, sigma=np.asarray(sigma, F32), out=out)
    x2 = rng.standard_normal((3, 17, 70, 1)).astype(F32)
    save('blur2d_s2', ref, x=x2, sigma=np.asarray(2.0, F32), out=npy(ne.layers.GaussianBlur(sigma=2.0)(T(x2))))
    x1 = rng.standard_normal((2, 50, 3)).astype(F32)
    save('blur1d_s1p2', ref, x=x1, sigma=np.asarray(1.2, F32), out=npy(ne.layers.GaussianBlur(sigma=1.2)(T(x1))))

    # separable_conv options: VALID, strides, dilations, single axis, unbatched
    k5 = rng.standard_normal(5).astype(F32)
    k4 = rng.standard_normal(4).astype(F32)
    xs = rng.standard_normal((2, 11, 13, 37, 3)).astype(F32)
    cases = [
        ('valid', dict(kernels=[T(k5)], padding='VALID', batched=True)),
        ('even_same', dict(kernels=[T(k4)], batched=True)),
        ('stride2', dict(kernels=[T(k5), T(k4), T(k5)], strides=2, batched=True)),
        ('dil2_axis1', dict(kernels=T(k5), axis=1, dilations=2, batched=True)),
        ('axes02', dict(kernels=[T(k4), T(k5)], axis=[0, 2], strides=[1, 3], batched=True)),
    ]
    for tag, kw in cases:
        out = npy(ne.utils.separable_conv(T(xs), **kw))
        save('sepconv_' + tag, ref, x=xs, k5=k5, k4=k4, out=out, kw=np.array(tag))
    out = npy(ne.utils.separable_conv(T(xs[0]), T(k5)))
    save('sepconv_unbatched', ref, x=xs[0], k5=k5, k4=k4, out=out, kw=np.array('unbatched'))


# ---------------------------------------------------------------------------------------
# PerlinNoise / GaussianNoise / draw_perlin_full / random_blur_rescale  (augment.py:65-218, layers.py:2305-2508)
# ---------------------------------------------------------------------------------------
def gen_noise():
    """The reference's own noise code on replayed draws: every tf.random call takes the next raw U[0, 1) or
    N(0, 1) array from tfshim.REPLAY, whose log (q0, q1, ... in call order) is stored with the output."""
    ref = ('reference neurite/tf/utils/augment.py:65-218 draw_perlin_full / random_blur_rescale, '
           'layers.py:2305-2508 GaussianNoise / PerlinNoise on tfshim (tf.random replayed from the stored draws)')
    tf = sys.modules['tensorflow']
    rng = np.random.default_rng(90)
    red = {'std': tf.math.reduce_std, 'max': tf.math.reduce_max}

    def run(name, fn, **meta):
        tfshim.REPLAY = tfshim.Replay(rng)
        out = npy(fn())
        q = {'q%d' % i: d for i, d in enumerate(tfshim.REPLAY.log)}
        save(name, ref, out=out, nq=np.array(len(q)), **q, **{k: np.asarray(v) for k, v in meta.items()})

    cases = [  # name, shape, levels (fwhm_min, fwhm_max), isotropic, reduce, axes, batched, featured
        ('perlin_2d_l1_std', (23, 31), ([2], [6]), False, 'std', None, False, False),
        ('perlin_2d_l3_max_iso', (20, 17, 2), ([1, 3, 5], [2, 8, 12]), True, 'max', -1, False, True),
        ('perlin_3d_l2_std_ax', (9, 12, 14, 3), ([2, 4], [4, 9]), False, 'std', -1, False, True),
        ('perlin_3d_l1_max_b2', (2, 10, 11, 13, 1), ([3], [7]), True, 'max', None, True, True),
        ('perlin_3d_l2_std_iso', (8, 9, 10), ([1, 2], [3, 5]), True, 'std', None, False, False),
    ]
    for name, shape, (lo, hi), iso, rd, axes, batched, featured in cases:
        run(name, lambda: ne.utils.augment.draw_perlin_full(
            list(shape), noise_min=0.05, noise_max=1.5, fwhm_min=lo, fwhm_max=hi, isotropic=iso, batched=batched,
            featured=featured, reduce=red[rd], axes=axes), shape=shape, fwhm_min=lo, fwhm_max=hi, isotropic=iso,
            reduce=rd, axes=-9 if axes is None else axes, batched=batched, featured=featured, noise_min=0.05,
            noise_max=1.5)

    x = rng.standard_normal((2, 12, 14, 3)).astype(F32)
    run('perlin_layer_2d_l2_std', lambda: ne.layers.PerlinNoise(fwhm_min=[2, 3], fwhm_max=[4, 6], axes=-1)(T(x)),
        x=x, fwhm_min=[2, 3], fwhm_max=[4, 6], isotropic=False, reduce='std', axes=-1, noise_min=0.01, noise_max=1.0)
    x3 = rng.standard_normal((2, 7, 9, 11, 1)).astype(F32)
    run('perlin_layer_3d_l1_max', lambda: ne.layers.PerlinNoise(shape=(7, 9, 11, 2), fwhm_min=3, fwhm_max=8,
                                                                   isotropic=True, reduce=tf.math.reduce_max)(T(x3)),
        x=x3, shape=(7, 9, 11, 2), fwhm_min=[3], fwhm_max=[8], isotropic=True, reduce='max', axes=-9,
        noise_min=0.01, noise_max=1.0)
    xb = rng.standard_normal((1, 15, 16, 2)).astype(F32)
    run('perlin_blur_rescale_2d_std', lambda: ne.utils.augment.random_blur_rescale(T(xb), std_min=0.5, std_max=2.5,
                                                                              batched=True),
        x=xb, std_min=0.5, std_max=2.5, isotropic=False, reduce='std')

    xg = (3 * rng.standard_normal((2, 6, 7, 8, 3))).astype(F32)
    for tag, kw in (('default', {}), ('noise_only', dict(noise_only=True)), ('absolute', dict(absolute=True)),
                    ('abs_only_ax1', dict(absolute=True, noise_only=True, axes=1))):
        kw = dict(noise_min=0.1, noise_max=0.2, **kw)
        run('gaussnoise_' + tag, lambda: ne.layers.GaussianNoise(**kw)(T(xg)), x=xg,
            **{k: v for k, v in kw.items()})


SYNTH_CASES = {  # name: (batch, labels drawn from, labels_to_image_new kwargs)
    'synth_3d_defaults_b2': (2, [0, 1, 2, 4], dict(
        labels_in=[0, 1, 2, 4], in_shape=(10, 12, 14), return_vel=True, return_def=True, return_mean=True,
        return_bias=True)),
    'synth_2d_dict_int_bg': (2, [0, 1, 2, 5, 7], dict(
        labels_in={0: 0, 1: 1, 2: 1, 5: 2, 7: 3}, labels_out={1: 1, 5: 2, 7: 2}, in_shape=(20, 22), num_chan=2,
        mean_min=[0, 0.2, 0.4, 0.6], mean_max=[0.1, 0.5, 0.6, 1.0], one_hot=False, crop_prob=1, crop_axes=1,
        zero_background=1, noise_max=0, gamma=0, slice_prob=1, return_mean=True)),
    'synth_3d_half_res_out': (1, [0, 1, 2, 3], dict(
        labels_in=[0, 1, 2, 3], in_shape=(12, 12, 16), out_shape=(10, 10, 12), half_res=True, warp_max=0, bias_max=0,
        normalize=False, gamma=0, crop_prob=1, crop_max=0.5, return_def=False, return_mean=True)),
    'synth_2d_list_gaps_gamma': (1, [0, 3, 5, 9], dict(
        labels_in=[0, 3, 5, 9], in_shape=(18, 16), crop_prob=1, crop_max=0.5, slice_prob=1, noise_max=0,
        zero_background=0, warp_max=0, return_mean=True, return_bias=True)),
    'synth_3d_noise_bg_nonorm': (1, [0, 1, 2], dict(
        labels_in=[0, 1, 2], in_shape=(8, 10, 12), zero_background=1, normalize=False, gamma=0, blur_max=0,
        bias_max=0, return_mean=True)),
}
CROP_CASES = {  # name: (input shape, dtype, RandomCrop kwargs)
    'crop_2d_bilateral_prob': ((2, 17, 23, 1), 'float32', dict(crop_min=0.1, crop_max=0.6, axis=2, prob=0.7,
                                                               bilateral=True)),
    'crop_3d_int_all_axes': ((1, 9, 11, 13, 2), 'int32', dict(crop_min=0.2, crop_max=0.4)),
    'crop_3d_axis_subset': ((2, 8, 10, 12, 1), 'float32', dict(crop_max=0.5, axis=[1, 3], prob=1)),
}


def gen_synth():
    """The reference's own labels_to_image_new, RandomCrop, draw_crop_mask and minmax_norm on replayed draws, with
    tools/vxmstub.py as voxelmorph (provenance 'contract' for the warp chain, as the st_* fixtures)."""
    import vxmstub
    vxmstub.install()
    rng = np.random.default_rng(123)
    ref = ('reference neurite/tf/models.py:920-1301 labels_to_image_new on tfshim + tools/vxmstub.py (voxelmorph '
           'warp chain: contract), tf.random replayed from the stored draws')

    class InputModel:
        def __init__(self, x):
            self.output, self.inputs = T(x), [T(x)]

    def log():
        return {'q%d' % i: d for i, d in enumerate(tfshim.REPLAY.log)}

    for name, (B, labs, kw) in SYNTH_CASES.items():
        x = rng.choice(np.asarray(labs), (B,) + tuple(kw['in_shape']) + (1,)).astype(np.int32)
        tfshim.REPLAY = tfshim.Replay(rng)
        args = dict(kw)
        args.pop('in_shape')
        outs = ne.models.labels_to_image_new(input_model=InputModel(x), **args)
        outs = outs if isinstance(outs, list) else [outs]
        q = log()
        save(name, ref, labels=x, kwargs=np.array(repr(kw)), nout=np.array(len(outs)),
             **{'out%d' % i: npy(o) for i, o in enumerate(outs)}, nq=np.array(len(q)), **q)

    ref_c = 'reference neurite/tf/layers.py:446-519 RandomCrop, utils/augment.py:221-287 on tfshim, draws replayed'
    for name, (shape, dt, kw) in CROP_CASES.items():
        x = (rng.integers(-5, 6, shape) if dt == 'int32' else rng.standard_normal(shape)).astype(dt)
        tfshim.REPLAY = tfshim.Replay(rng)
        out = npy(ne.layers.RandomCrop(**kw)(T(x)))
        q = log()
        save(name, ref_c, x=x, out=out, kwargs=np.array(repr(kw)), nq=np.array(len(q)), **q)
    xm = rng.standard_normal((3, 7, 5)).astype(F32)
    tfshim.REPLAY = tfshim.Replay(rng)
    m = npy(ne.utils.augment.draw_crop_mask(T(xm), crop_min=0.3, crop_max=0.3, axis=None, prob=1))
    q = log()
    save('crop_mask_fixed_prop', ref_c, x=xm, out=m, kwargs=np.array(repr(dict(crop_min=0.3, crop_max=0.3))),
         nq=np.array(len(q)), **q)

    ref_m = 'reference neurite/tf/utils/utils.py:953-968 minmax_norm on tfshim'
    for name, shape, axis in (('minmax_all', (2, 9, 11, 3), None), ('minmax_trailing', (3, 8, 7, 2), (1, 2, 3))):
        x = (2 * rng.standard_normal(shape) + 1).astype(F32)
        save(name, ref_m, x=x, out=npy(ne.utils.minmax_norm(T(x), axis=axis)), axis=np.array(repr(axis)))
    xc = np.full((2, 4, 5), 3.0, F32)
    save('minmax_constant', ref_m, x=xc, out=npy(ne.utils.minmax_norm(T(xc))), axis=np.array('None'))


_ALL3 = dict(aff_shift=3, aff_rotate=20, aff_scale=0.2, aff_shear=0.1)
AFFSYNTH_CASES = {  # name: (batch, labels drawn from, labels_to_image_new kwargs)
    'affsynth_3d_uniform_all': (2, [0, 1, 2, 4], dict(
        labels_in=[0, 1, 2, 4], in_shape=(10, 12, 14), return_aff=True, return_def=True, **_ALL3)),
    'affsynth_3d_normal_all': (2, [0, 1, 2, 3], dict(
        labels_in=[0, 1, 2, 3], in_shape=(10, 12, 14), aff_shift=2, aff_rotate=15, aff_scale=0.3, aff_shear=0.1,
        aff_normal_shift=True, aff_normal_rotate=True, aff_normal_scale=True, aff_normal_shear=True, bias_max=0,
        return_aff=True)),
    'affsynth_2d_shift': (2, [0, 1, 2], dict(labels_in=[0, 1, 2], in_shape=(20, 22), aff_shift=4, return_aff=True)),
    'affsynth_2d_rotate_normal': (2, [0, 1, 2], dict(
        labels_in=[0, 1, 2], in_shape=(20, 22), aff_rotate=30, aff_normal_rotate=True, return_aff=True)),
    'affsynth_2d_scale_normal': (2, [0, 1, 2], dict(
        labels_in=[0, 1, 2], in_shape=(18, 16), aff_scale=0.25, aff_normal_scale=True, return_aff=True)),
    'affsynth_3d_shear': (2, [0, 1, 2], dict(labels_in=[0, 1, 2], in_shape=(10, 12, 14), aff_shear=0.2,
                                             return_aff=True)),
    'affsynth_3d_flip': (2, [0, 1, 2, 3], dict(labels_in=[0, 1, 2, 3], in_shape=(10, 12, 14), aff_rotate=10,
                                               axes_flip=True, return_aff=True)),
    'affsynth_3d_swap_iso': (2, [0, 1, 2, 3], dict(labels_in=[0, 1, 2, 3], in_shape=(10, 10, 10), aff_shift=2,
                                                   axes_swap=True, axes_flip=True, return_aff=True)),
    'affsynth_3d_half_res_out': (2, [0, 1, 2, 3], dict(
        labels_in=[0, 1, 2, 3], in_shape=(12, 12, 16), out_shape=(10, 10, 12), half_res=True, aff_rotate=15,
        aff_scale=0.1, bias_max=0, return_aff=True)),
    'affsynth_2d_out_smaller': (2, [0, 1, 2, 5], dict(
        labels_in=[0, 1, 2, 5], in_shape=(20, 24), out_shape=(16, 18), aff_shift=2, aff_rotate=25, aff_scale=0.15,
        aff_shear=0.1, one_hot=False, return_aff=True)),
    'affsynth_3d_nowarp': (2, [0, 1, 2, 3], dict(labels_in=[0, 1, 2, 3], in_shape=(10, 12, 14), warp_max=0,
                                                 return_aff=True, **_ALL3)),
}


def gen_affsynth():
    """The reference's own labels_to_image_new with random affine, flip and swap augmentation, on replayed draws,
    with tools/vxmstub.py as voxelmorph (provenance 'contract').  Each fixture also stores the [B, N, N+1] matrix
    the reference hands to AffineToDenseShift ('trans')."""
    import vxmstub
    vxmstub.install()
    rng = np.random.default_rng(321)
    ref = ('reference neurite/tf/models.py:920-1301 labels_to_image_new on tfshim + tools/vxmstub.py (voxelmorph '
           'affine draw, matrices and warp chain: contract), tf.random replayed from the stored draws')

    class InputModel:
        def __init__(self, x):
            self.output, self.inputs = T(x), [T(x)]

    for name, (B, labs, kw) in AFFSYNTH_CASES.items():
        x = rng.choice(np.asarray(labs), (B,) + tuple(kw['in_shape']) + (1,)).astype(np.int32)
        tfshim.REPLAY = tfshim.Replay(rng)
        vxmstub.LAST_TRANS.clear()
        args = dict(kw)
        args.pop('in_shape')
        outs = ne.models.labels_to_image_new(input_model=InputModel(x), **args)
        outs = outs if isinstance(outs, list) else [outs]
        q = {'q%d' % i: d for i, d in enumerate(tfshim.REPLAY.log)}
        assert len(vxmstub.LAST_TRANS) == 1
        save(name, ref, labels=x, kwargs=np.array(repr(kw)), nout=np.array(len(outs)), trans=vxmstub.LAST_TRANS[0],
             **{'out%d' % i: npy(o) for i, o in enumerate(outs)}, nq=np.array(len(q)), **q)


if __name__ == '__main__':
    only = sys.argv[2:]
    for fn in (gen_interpn, gen_resize, gen_spatial_transformer, gen_dice, gen_lc3d, gen_lc3d_impl, gen_mi, gen_blur,
               gen_noise, gen_synth, gen_affsynth):
        if not only or fn.__name__[4:] in only:
            fn()
    tot = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print('total %.1f KB in %s' % (tot / 1024, OUT))
