"""
GPU parity tests (run on an H100: `pytest -m gpu`).  Everything goes through the public
python API -> ctypes -> the C ABI of libneurite_b200.so.  Checked against
  * tests/golden/*.npz   (outputs of the reference's own source, see tools/gen_golden.py)
  * the numpy oracle      (oracle/, same seeded inputs, incl. BASELINE.json's full 160x192x224)
  * size-independent properties (identity warp, slab == whole, tile path == gather path).

Tolerances: interpolation family is BIT-EXACT (np.array_equal) -- the kernels round every
multiply/add separately like the reference's unfused TF ops.  Reductions (Dice, CCE, LC3D)
use rtol 1e-5 (north_star), because TF's reduction order is unspecified.
"""

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import interp as ointerp, lc3d as olc3d, metrics as ometrics

pytestmark = pytest.mark.gpu
F32 = np.float32


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _fill(g):
    f = float(g['fill'])
    return None if np.isnan(f) else f


@pytest.fixture(scope='module')
def ne(cuda):
    import neurite_b200
    return neurite_b200


# ------------------------------------------------------------------ golden: interpn / resize / warp
@pytest.mark.parametrize('name', golden_names('interpn_'))
def test_interpn_golden(ne, name):
    g = load_golden(name)
    loc = dev(g['loc'])
    if '_list_' in name:
        loc = [loc[..., d] for d in range(loc.shape[-1])]
    fill = _fill(g) if 'fill' in g.files else None
    out = ne.utils.interpn(dev(g['vol']), loc, str(g['method']), fill).cpu().numpy()
    assert out.shape == g['out'].shape
    np.testing.assert_array_equal(out, g['out'])


@pytest.mark.parametrize('name', golden_names('resize_'))
def test_resize_golden(ne, name):
    g = load_golden(name)
    z = g['zoom']
    z = float(z) if z.ndim == 0 else [float(v) for v in z]
    if isinstance(z, float) and z.is_integer():
        z = int(z)
    if name.startswith('resize_layer'):
        out = ne.layers.Resize(z, interp_method=str(g['method']))(dev(g['x']))
    else:
        out = ne.utils.resize(dev(g['vol']), z, interp_method=str(g['method']))
    np.testing.assert_array_equal(out.cpu().numpy(), g['out'])


@pytest.mark.parametrize('name', golden_names('st_'))
def test_spatial_transformer_golden(ne, name):
    g = load_golden(name)
    lay = ne.layers.SpatialTransformer(interp_method=str(g['method']), fill_value=_fill(g))
    out = lay([dev(g['vol']), dev(g['flow'])]).cpu().numpy()
    np.testing.assert_array_equal(out, g['out'])


# ------------------------------------------------------------------ tiled (TMA) path vs oracle
def _rand_case(shape, amp, seed, smooth=False, channels=1):
    rng = np.random.default_rng(seed)
    vol = rng.standard_normal((1,) + shape + (channels,)).astype(F32)
    flow = rng.uniform(-amp, amp, (1,) + shape + (3,)).astype(F32)
    return vol, flow


@pytest.mark.parametrize('shape,amp,halo', [((20, 40, 64), 3.0, 3), ((17, 24, 36), 6.0, 4), ((9, 16, 32), 2.0, 5),
                                            ((33, 18, 100), 3.0, 0), ((40, 48, 96), 9.0, 8), ((16, 16, 36), 5.0, 4),
                                            ((12, 20, 32), 4.0, 4)])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', -2.5), ('nearest', 0.0)])
@pytest.mark.parametrize('C', [1, 2])
def test_warp_box_tile_bit_exact(ne, monkeypatch, C, shape, amp, halo, method, fill):
    """TMA box-tile warp kernel: C = 1 on 8x8x32 tiles with the halo (3, 4, 6, 8) chosen from `halo`, C = 2 on
    4x8x32 tiles with (x, channel) as one TMA dimension; flows inside, across and far outside the staged box; equal to
    the oracle and to the generic gather kernel."""
    vol, flow = _rand_case(shape, amp, seed=2, channels=C)
    flow[0, 0, 0, :4] = [[0, 0, 0], [0.5, 1.5, -0.5], [-40, 50, 3], [1, 1, 1]]
    ref = ointerp.spatial_transformer(vol, flow, method, 'ij', fill)
    lay = ne.layers.SpatialTransformer(interp_method=method, fill_value=fill, halo=halo)
    out = lay([dev(vol), dev(flow)]).cpu().numpy()
    np.testing.assert_array_equal(out, ref)
    monkeypatch.setenv('NRT_WARP_TILE', '0')                 # generic gather kernel
    out2 = lay([dev(vol), dev(flow)]).cpu().numpy()
    np.testing.assert_array_equal(out2, ref)


@pytest.mark.parametrize('C', [2, 3, 4, 8, 12, 16, 32])
@pytest.mark.parametrize('shape,amp', [((20, 24, 32), 3.0), ((11, 13, 52), 6.0), ((40, 18, 100), 2.5)])
def test_warp_march_kernel_multichannel_bit_exact(ne, monkeypatch, C, shape, amp):
    """z-marching ring kernel (nrt_warp_march.cu): every channel count it is built for, ragged tiles, flows
    inside and far outside the staged window, one and two quads per thread, forced z segmentations (down to one
    output plane per segment); C = 2 takes the box-tile kernel."""
    rng = np.random.default_rng(C * 100 + shape[0])
    vol = rng.standard_normal((2,) + shape + (C,)).astype(F32)
    flow = rng.uniform(-amp, amp, (2,) + shape + (3,)).astype(F32)
    flow[1] += np.array([1.2, -0.7, 2.1], dtype=F32)
    flow[0, 0, 0, :3] = [[0, 0, 0], [-40, 50, 3], [0.5, 1.5, -0.5]]
    vol[1, 2:5, 3:7] = 0.0                                   # exact zeros of either sign: the packed a*b = fma(a, b, -0)
    vol[1, 3, 4:6] = -0.0                                    # must give the scalar chain's sign of zero
    dv, df = dev(vol), dev(flow)
    for method, fill in (('linear', None), ('linear', -1.5), ('nearest', 0.0)):
        ref = ointerp.spatial_transformer(vol, flow, method, 'ij', fill)
        lay = ne.layers.SpatialTransformer(interp_method=method, fill_value=fill)
        for env in ({}, {'NRT_MARCH_NSEG': '3'}, {'NRT_MARCH_NSEG': '40'}):
            monkeypatch.delenv('NRT_MARCH_NSEG', raising=False)
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            out = lay([dv, df]).cpu().numpy()
            np.testing.assert_array_equal(out, ref)
            np.testing.assert_array_equal(np.signbit(out), np.signbit(ref))


def test_warp_box_follows_smooth_flow(ne, monkeypatch):
    """large smooth displacement: the staged box follows the flow (and results never depend on it)"""
    rng = np.random.default_rng(21)
    S = (24, 32, 64)
    vol = rng.standard_normal((2,) + S + (1,)).astype(F32)
    base = np.array([9.3, -7.6, 11.2], dtype=F32)
    flow = (base + rng.uniform(-1.5, 1.5, (2,) + S + (3,))).astype(F32)
    ref = ointerp.spatial_transformer(vol, flow)
    for follow in ('1', '0'):
        monkeypatch.setenv('NRT_WARP_FOLLOW', follow)
        out = ne.layers.SpatialTransformer()([dev(vol), dev(flow)]).cpu().numpy()
        np.testing.assert_array_equal(out, ref)


def test_warp_batch_and_channels(ne):
    rng = np.random.default_rng(5)
    for C in (1, 2, 3, 4, 16):
        for S, amp in (((12, 16, 32), 3.0), ((9, 13, 68), 5.0)):
            vol = rng.standard_normal((3,) + S + (C,)).astype(F32)
            flow = rng.uniform(-amp, amp, (3,) + S + (3,)).astype(F32)
            flow[1] += np.array([6.2, -5.1, 9.7], dtype=F32)              # coherent shift: box re-staging
            for method, fill in (('linear', None), ('linear', 1.5), ('nearest', 0.0)):
                ref = ointerp.spatial_transformer(vol, flow, method, 'ij', fill)
                out = ne.layers.SpatialTransformer(interp_method=method, fill_value=fill)([dev(vol), dev(flow)]).cpu().numpy()
                np.testing.assert_array_equal(out, ref)
    # xy indexing swaps the first two shift channels
    vol = rng.standard_normal((1, 8, 9, 12, 1)).astype(F32)
    flow = rng.uniform(-2, 2, (1, 8, 9, 12, 3)).astype(F32)
    ref = ointerp.spatial_transformer(vol, flow, indexing='xy')
    out = ne.layers.SpatialTransformer(indexing='xy')([dev(vol), dev(flow)]).cpu().numpy()
    np.testing.assert_array_equal(out, ref)


def test_warp_full_size_cfg2_bit_exact_vs_oracle(ne):
    """BASELINE.json configs[1]: 160x192x224 fp32, random dense flow (SURVEY.md 8d seeds)."""
    S = (160, 192, 224)
    vol = np.random.default_rng(0).standard_normal((1,) + S + (1,)).astype(F32)
    flow = np.random.default_rng(1).uniform(-3, 3, (1,) + S + (3,)).astype(F32)
    dv, df = dev(vol), dev(flow)
    out = ne.layers.SpatialTransformer()([dv, df])
    ref = ointerp.spatial_transformer(vol, flow)
    np.testing.assert_array_equal(out.cpu().numpy(), ref)
    # identity warp returns the input bit for bit
    ident = ne.layers.SpatialTransformer()([dv, torch.zeros_like(df)])
    assert torch.equal(ident, dv)
    # the reference's in-repo usage: nearest + fill 0 on label maps (models.py:806-809)
    lab = np.random.default_rng(2).integers(0, 16, vol.shape).astype(F32)
    out = ne.layers.SpatialTransformer(interp_method='nearest', fill_value=0)([dev(lab), df]).cpu().numpy()
    np.testing.assert_array_equal(out, ointerp.spatial_transformer(lab, flow, 'nearest', 'ij', 0))


def test_warp_slabs_equal_whole(ne):
    """z-slab sharding arithmetic on one GPU: each 'rank' warps its slab against only the
    source window it would hold; concatenation == whole-volume warp, bit for bit."""
    from neurite_b200 import dist as nd, utils
    rng = np.random.default_rng(7)
    S = (24, 20, 32)
    for C, world_list in ((1, (2, 3, 8)), (2, (3,)), (16, (2,))):
        _check_slabs(nd, utils, rng, S, C, world_list)
    vol = dev(rng.standard_normal((2,) + S + (1,)).astype(F32))
    flow = dev(rng.uniform(-3, 3, (2,) + S + (3,)).astype(F32))
    # a window that is too small is reported, not silently wrong
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    utils._warp_batched(vol[:, 8:12].contiguous(), flow[:, 8:12].contiguous() * 4, src_z0=8, full_s0=S[0], out_z0=8,
                        err_flag=err)
    assert int(err.item()) == 1


def _check_slabs(nd, utils, rng, S, C, world_list):
    vol = dev(rng.standard_normal((2,) + S + (C,)).astype(F32))
    flow = dev(rng.uniform(-3, 3, (2,) + S + (3,)).astype(F32))
    whole = utils._warp_batched(vol, flow)
    for world in world_list:
        parts = []
        for r in range(world):
            z0, nz = nd.slab_bounds(S[0], world, r)
            h = nd.required_halo(flow[:, z0:z0 + nz])
            lo, hi = nd.source_window(z0, nz, h, S[0])
            err = torch.zeros(1, dtype=torch.int32, device='cuda')
            parts.append(utils._warp_batched(vol[:, lo:hi].contiguous(), flow[:, z0:z0 + nz].contiguous(),
                                             src_z0=lo, full_s0=S[0], out_z0=z0, err_flag=err))
            assert int(err.item()) == 0
        assert torch.equal(torch.cat(parts, 1), whole)


def test_resize_full_size_and_slabs(ne):
    from neurite_b200 import utils
    rng = np.random.default_rng(8)
    x = rng.standard_normal((1, 80, 96, 112, 3)).astype(F32)           # half-res flow -> full res (models.py:803-804)
    out = ne.layers.Resize(2)(dev(x))
    assert tuple(out.shape) == (1, 160, 192, 224, 3)
    ref = ointerp.resize_layer(x, 2)
    np.testing.assert_array_equal(out.cpu().numpy(), ref)
    x3 = dev(np.concatenate([x, x[:, ::-1].copy(), x * 0.5], 0))
    out3 = ne.layers.Resize(2)(x3)
    assert torch.equal(out3[0], out[0]) and torch.equal(out3[2], ne.layers.Resize(2)(x3[2:3])[0])
    np.testing.assert_array_equal(out3[1].cpu().numpy(), ointerp.resize_layer(x[:, ::-1], 2)[0])
    a = utils._resize_batched(dev(x), [2, 2, 2], 'linear', out_z0=0, out_n0=70)
    b = utils._resize_batched(dev(x), [2, 2, 2], 'linear', out_z0=70, out_n0=90)
    assert torch.equal(torch.cat([a, b], 1), out)


# ------------------------------------------------------------------ Dice / CCE
@pytest.mark.parametrize('name', ['dice_soft_default', 'dice_soft_laplace_weights', 'dice_soft_normalize',
                                  'dice_hard_prob', 'dice_hard_max_label', 'dice_soft_disjoint_L5'])
def test_dice_golden(ne, name):
    import warnings
    g = load_golden(name)
    kw = {}
    if name == 'dice_soft_laplace_weights':
        kw = dict(weights=g['weights'], laplace_smoothing=0.1)
    elif name == 'dice_soft_normalize':
        kw = dict(normalize=True)
    elif name == 'dice_hard_prob':
        kw = dict(dice_type='hard', input_type='prob')
    elif name == 'dice_hard_max_label':
        kw = dict(dice_type='hard', input_type='max_label', nb_labels=int(g['nb_labels']))
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        d = ne.losses.Dice(**kw)
        t, p = dev(g['y_true']), dev(g['y_pred'])
        np.testing.assert_allclose(d.dice(t, p).cpu().numpy(), g['dice'], rtol=1e-5, atol=1e-7)
        for k, fn in (('loss', d.loss), ('mean_dice', d.mean_dice), ('mean_loss', d.mean_loss)):
            if k in g.files:
                np.testing.assert_allclose(fn(t, p).cpu().numpy(), g[k], rtol=1e-5, atol=1e-7)


def test_dice_range_check_and_properties(ne):
    g = load_golden('dice_range_error')
    with pytest.raises(ne.metrics.InvalidArgumentError, match='value outside range'):
        ne.losses.Dice().dice(dev(g['y_true']), dev(g['y_pred']))
    ne.losses.Dice(check_input_limits=False).dice(dev(g['y_true']), dev(g['y_pred']))
    nan = g['y_pred'].copy()
    nan[0, 0, 0, 0, 0] = np.nan
    with pytest.raises(ne.metrics.InvalidArgumentError):
        ne.losses.Dice().dice(dev(g['y_true']), dev(nan))
    rng = np.random.default_rng(0)
    for L in (1, 3, 4, 5, 8, 16, 20, 64):
        lab = rng.integers(0, L, (2, 7, 9, 11))
        t = np.eye(L, dtype=F32)[lab]
        p = rng.uniform(0, 1, t.shape).astype(F32)
        d = ne.losses.Dice()
        one = d.dice(dev(t), dev(t)).cpu().numpy()
        present = np.stack([[np.any(lab[b] == l) for l in range(L)] for b in range(2)])
        np.testing.assert_array_equal(one, present.astype(F32))          # Dice(x,x) = 1, absent label 0/0 -> 0
        a = d.dice(dev(t), dev(p)).cpu().numpy()
        np.testing.assert_allclose(a, d.dice(dev(p), dev(t)).cpu().numpy(), rtol=1e-6)     # symmetric
        np.testing.assert_allclose(a, ometrics.Dice().dice(t, p), rtol=1e-5, atol=1e-7)


def test_dice_cfg3_scale_vs_oracle(ne):
    """cfg 3 shape per batch item (16 labels on 160x192x224), batch 1 to keep the oracle in seconds."""
    rng = np.random.default_rng(3)
    S, L = (160, 192, 224), 16
    lab = rng.integers(0, L, (1,) + S)
    t = torch.nn.functional.one_hot(torch.from_numpy(lab).cuda(), L).float()
    logits = torch.randn((1,) + S + (L,), device='cuda', generator=torch.Generator('cuda').manual_seed(1))
    p = torch.softmax(logits, -1)
    d = ne.losses.Dice()
    out = d.loss(t, p).cpu().numpy()
    tt, pp = t.cpu().numpy(), p.cpu().numpy()
    ref = ometrics.Dice().loss(tt, pp)
    np.testing.assert_allclose(out, ref, rtol=1e-5)
    np.testing.assert_allclose(float(d.mean_loss(t, p)), ometrics.Dice().mean_loss(tt, pp), rtol=1e-5)
    c = ne.losses.CategoricalCrossentropy(label_weights=np.linspace(0.5, 2, L))
    np.testing.assert_allclose(float(c.loss(t, p)),
                               ometrics.categorical_crossentropy(tt, pp, np.linspace(0.5, 2, L).astype(F32)), rtol=1e-5)


@pytest.mark.parametrize('name', ['cce_label_weights', 'cce_plain'])
def test_cce_golden(ne, name):
    g = load_golden(name)
    lw = g['label_weights'] if 'label_weights' in g.files else None
    c = ne.losses.CategoricalCrossentropy(label_weights=lw)
    np.testing.assert_allclose(float(c.loss(dev(g['y_true']), dev(g['y_pred']))), g['loss'], rtol=1e-5)


def test_cce_variants_vs_oracle(ne):
    """every lanes-per-row instantiation (C = 4 .. 128), the row kernel (C = 2, 3, 5); 2 x 37 x 41 rows: a ragged
    last pass of the four-rows-per-thread loop"""
    rng = np.random.default_rng(11)
    for C in (2, 3, 4, 5, 8, 16, 32, 64, 128):
        t = np.eye(C, dtype=F32)[rng.integers(0, C, (2, 37, 41) if C in (4, 16) else (2, 6, 7))]
        p = rng.uniform(0.01, 1, t.shape).astype(F32)
        lw = rng.uniform(0.5, 2, C).astype(F32)
        sw = rng.uniform(0.5, 2, t.shape[:-1]).astype(F32)
        for kw in (dict(), dict(label_weights=lw), dict(label_weights=lw, sample_weight=sw),
                   dict(from_logits=True), dict(label_smoothing=0.1), dict(reduction='sum')):
            okw = dict(kw)
            sample = okw.pop('sample_weight', None)
            ref = ometrics.categorical_crossentropy(t, p, sample_weight=sample, **okw)
            ckw = {k: v for k, v in okw.items()}
            c = ne.losses.CategoricalCrossentropy(**ckw)
            out = c(dev(t), dev(p), sample_weight=None if sample is None else dev(sample))
            np.testing.assert_allclose(float(out), ref, rtol=2e-5)
        per = ne.losses.CategoricalCrossentropy(reduction='none')(dev(t), dev(p)).cpu().numpy()
        np.testing.assert_allclose(per, ometrics.categorical_crossentropy(t, p, reduction='none'), rtol=2e-5, atol=1e-6)
    one = np.eye(3, dtype=F32)[[0, 1, 2, 1]][None]
    np.testing.assert_allclose(float(ne.losses.CategoricalCrossentropy()(dev(one), dev(one))), -np.log(1 - 1e-7),
                               rtol=1e-3, atol=2e-7)


# ------------------------------------------------------------------ LocallyConnected3D
@pytest.mark.parametrize('generic', [False, True])
@pytest.mark.parametrize('name', [n for n in golden_names('lc3d_') if 'impl_idx' not in n])
def test_lc3d_golden(ne, monkeypatch, name, generic):
    if generic:
        monkeypatch.setenv('NRT_LC3D_GENERIC', '1')
    g = load_golden(name)
    fmt = str(g['data_format'])
    use_bias = bool(g['bias'].size)
    lay = ne.layers.LocallyConnected3D(int(g['filters']), tuple(int(k) for k in g['kernel_size']),
                                       strides=tuple(int(s) for s in g['strides']), data_format=fmt, use_bias=use_bias)
    lay.build(g['x'].shape)
    assert tuple(lay.kernel.shape) == g['kernel'].shape
    with torch.no_grad():
        lay.kernel.copy_(torch.from_numpy(g['kernel']))
        if use_bias:
            lay.bias.copy_(torch.from_numpy(g['bias']))
    lay.cuda()
    out = lay(dev(g['x'])).detach().cpu().numpy()
    assert out.shape == g['out'].shape
    np.testing.assert_allclose(out, g['out'], rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize('patch', ['1', '0'])
def test_lc3d_vs_oracle_batches_activations_and_sharding(ne, monkeypatch, patch):
    """batch 11 = passes of 8 + 2 + 1 items: the TMA-patch kernel (batch > 1) and the register-gather kernel are
    bit-identical, all within 1e-5 of the oracle."""
    from neurite_b200.layers import local_conv3d
    monkeypatch.setenv('NRT_LC3D_PATCH', patch)
    rng = np.random.default_rng(13)
    x = rng.standard_normal((11, 8, 9, 10, 16)).astype(F32)
    O = (6, 7, 8)
    kernel = (rng.standard_normal((int(np.prod(O)), 27 * 16, 16)) * 0.05).astype(F32)
    bias = rng.standard_normal(O + (16,)).astype(F32)
    for act in (None, 'relu', 'tanh', 'sigmoid'):
        ref = olc3d.locally_connected_3d(x, kernel, bias, (3, 3, 3), activation=act, literal=False)
        out = local_conv3d(dev(x), dev(kernel), dev(bias), (3, 3, 3), (1, 1, 1), O, activation=act).cpu().numpy()
        np.testing.assert_allclose(out, ref, rtol=1e-5, atol=2e-5)
    # (the quad-per-lane kernels share one summation order; the row kernels are compared in their own test)
    monkeypatch.setenv('NRT_LC3D_ROWS', '0')
    out = local_conv3d(dev(x), dev(kernel), dev(bias), (3, 3, 3), (1, 1, 1), O, activation='sigmoid').cpu().numpy()
    monkeypatch.setenv('NRT_LC3D_PATCH', '0')
    gather = local_conv3d(dev(x), dev(kernel), dev(bias), (3, 3, 3), (1, 1, 1), O, activation='sigmoid').cpu().numpy()
    np.testing.assert_array_equal(out, gather)
    monkeypatch.setenv('NRT_LC3D_PATCH', patch)
    # strides > 1 and a ragged weight block (F * Cout / 4 not a multiple of 32): patch origin = position * stride
    xs = rng.standard_normal((4, 9, 8, 11, 4)).astype(F32)
    Os = (4, 3, 5)
    ks = (rng.standard_normal((int(np.prod(Os)), 2 * 3 * 2 * 4, 4)) * 0.1).astype(F32)
    refs = olc3d.locally_connected_3d(xs, ks, None, (2, 3, 2), strides=(2, 2, 2), literal=False)
    outs = local_conv3d(dev(xs), dev(ks), None, (2, 3, 2), (2, 2, 2), Os).cpu().numpy()
    np.testing.assert_allclose(outs, refs, rtol=1e-5, atol=2e-5)
    # position sharding: two ranks each own half of the positions AND of the weights
    ref = olc3d.locally_connected_3d(x, kernel, bias, (3, 3, 3), literal=False).reshape(11, -1, 16)
    P = kernel.shape[0]
    h = P // 2 + 3
    a = local_conv3d(dev(x), dev(kernel[:h]), dev(bias.reshape(-1, 16)[:h]), (3, 3, 3), (1, 1, 1), O, p0=0, p_count=h)
    b = local_conv3d(dev(x), dev(kernel[h:]), dev(bias.reshape(-1, 16)[h:]), (3, 3, 3), (1, 1, 1), O, p0=h, p_count=P - h)
    np.testing.assert_allclose(torch.cat([a, b], 1).cpu().numpy(), ref, rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize('rows', ['1', '0'])
def test_lc3d_row_kernel_vs_oracle(ne, monkeypatch, rows):
    """batch 13 = passes of 8 + 4 + 1 items: the pass of 8 through the row kernel (lanes own patch rows and all 16
    channels, two warps x four items per position) or the quad-per-lane patch kernel, against the oracle; bias,
    activations, a ragged patch (F = 20 < 32 rows), F = 48, strides 2, position shards"""
    from neurite_b200.layers import local_conv3d
    monkeypatch.setenv('NRT_LC3D_ROWS', rows)
    rng = np.random.default_rng(113)
    x = rng.standard_normal((13, 8, 9, 10, 16)).astype(F32)
    O = (6, 7, 8)
    kernel = (rng.standard_normal((int(np.prod(O)), 27 * 16, 16)) * 0.05).astype(F32)
    bias = rng.standard_normal(O + (16,)).astype(F32)
    for act in (None, 'relu', 'sigmoid'):
        ref = olc3d.locally_connected_3d(x, kernel, bias, (3, 3, 3), activation=act, literal=False)
        out = local_conv3d(dev(x), dev(kernel), dev(bias), (3, 3, 3), (1, 1, 1), O, activation=act).cpu().numpy()
        np.testing.assert_allclose(out, ref, rtol=1e-5, atol=2e-5)
    out = local_conv3d(dev(x), dev(kernel), None, (3, 3, 3), (1, 1, 1), O).cpu().numpy()
    np.testing.assert_allclose(out, olc3d.locally_connected_3d(x, kernel, None, (3, 3, 3), literal=False), rtol=1e-5, atol=2e-5)
    for ks, st, Cin, shp in (((1, 1, 5), (1, 1, 1), 4, (3, 4, 9)), ((2, 3, 2), (2, 2, 2), 4, (9, 8, 11)), ((2, 2, 2), (1, 2, 1), 8, (5, 6, 4))):
        xs = rng.standard_normal((12,) + shp + (Cin,)).astype(F32)
        Os = tuple((shp[d] - ks[d]) // st[d] + 1 for d in range(3))
        kk = (rng.standard_normal((int(np.prod(Os)), int(np.prod(ks)) * Cin, 16)) * 0.1).astype(F32)
        bb = rng.standard_normal(Os + (16,)).astype(F32)
        refs = olc3d.locally_connected_3d(xs, kk, bb, ks, strides=st, activation='tanh', literal=False)
        outs = local_conv3d(dev(xs), dev(kk), dev(bb), ks, st, Os, activation='tanh').cpu().numpy()
        np.testing.assert_allclose(outs, refs, rtol=1e-5, atol=2e-5)
    # position sharding with the same kernels
    ref = olc3d.locally_connected_3d(x, kernel, bias, (3, 3, 3), literal=False).reshape(13, -1, 16)
    P = kernel.shape[0]
    h = P // 2 + 3
    a = local_conv3d(dev(x), dev(kernel[:h]), dev(bias.reshape(-1, 16)[:h]), (3, 3, 3), (1, 1, 1), O, p0=0, p_count=h)
    b = local_conv3d(dev(x), dev(kernel[h:]), dev(bias.reshape(-1, 16)[h:]), (3, 3, 3), (1, 1, 1), O, p0=h, p_count=P - h)
    np.testing.assert_allclose(torch.cat([a, b], 1).cpu().numpy(), ref, rtol=1e-5, atol=2e-5)


@pytest.mark.parametrize('rows', ['1', '0'])
def test_lc3d_batch8_shared_weights_equal_conv3d(ne, monkeypatch, rows):
    """cfg 4 geometry, batch 8, many positions per CTA (22^3 positions over 132 CTAs: every ring slot is reused many
    times): with position-shared weights the layer must equal a plain conv3d"""
    monkeypatch.setenv('NRT_LC3D_ROWS', rows)
    rng = np.random.default_rng(19)
    x = torch.from_numpy(rng.standard_normal((8, 24, 24, 24, 16)).astype(F32)).cuda()
    w = torch.from_numpy((rng.standard_normal((3, 3, 3, 16, 16)) * 0.1).astype(F32)).cuda()
    P = 22 ** 3
    kernel = w.reshape(1, 432, 16).expand(P, 432, 16).contiguous()
    from neurite_b200.layers import local_conv3d
    out = local_conv3d(x, kernel, None, (3, 3, 3), (1, 1, 1), (22, 22, 22))
    torch.backends.cudnn.allow_tf32 = False
    ref = torch.nn.functional.conv3d(x.permute(0, 4, 1, 2, 3), w.permute(4, 3, 0, 1, 2)).permute(0, 2, 3, 4, 1)
    np.testing.assert_allclose(out.cpu().numpy(), ref.cpu().numpy(), rtol=1e-4, atol=1e-4)


def test_lc3d_shared_weights_equal_conv3d_cfg4_shape(ne):
    """cfg 4 geometry (3^3 kernel, 16->16) on a 24^3 crop: with position-shared weights the
    layer must equal a plain conv3d (independent implementation: cuDNN through torch)."""
    rng = np.random.default_rng(17)
    x = torch.from_numpy(rng.standard_normal((2, 24, 24, 24, 16)).astype(F32)).cuda()
    w = torch.from_numpy((rng.standard_normal((3, 3, 3, 16, 16)) * 0.1).astype(F32)).cuda()
    P = 22 ** 3
    kernel = w.reshape(1, 432, 16).expand(P, 432, 16).contiguous()
    from neurite_b200.layers import local_conv3d
    out = local_conv3d(x, kernel, None, (3, 3, 3), (1, 1, 1), (22, 22, 22))
    torch.backends.cudnn.allow_tf32 = False
    ref = torch.nn.functional.conv3d(x.permute(0, 4, 1, 2, 3), w.permute(4, 3, 0, 1, 2)).permute(0, 2, 3, 4, 1)
    np.testing.assert_allclose(out.cpu().numpy(), ref.cpu().numpy(), rtol=1e-4, atol=1e-4)


def test_warp_host_pipeline_matches_device_path(ne):
    rng = np.random.default_rng(31)
    vol = torch.from_numpy(rng.standard_normal((5, 12, 16, 32, 1)).astype(F32)).pin_memory()
    flow = torch.from_numpy(rng.uniform(-3, 3, (5, 12, 16, 32, 3)).astype(F32)).pin_memory()
    lay = ne.layers.SpatialTransformer()
    ref = lay([vol.cuda(), flow.cuda()]).cpu()
    for chunk in (1, 2, 5):
        out = lay.call_host([vol, flow], chunk=chunk)
        assert not out.is_cuda and torch.equal(out, ref)
    buf = torch.empty_like(ref).pin_memory()
    assert lay.call_host([vol, flow], out=buf) is buf and torch.equal(buf, ref)


def test_empty_and_degenerate_inputs(ne):
    """empty / size-1 inputs behave like the reference's gather (no launch, right shapes)."""
    vol = torch.randn(4, 5, 6, 2, device='cuda')
    out = ne.utils.interpn(vol, torch.zeros((0, 3), device='cuda'))
    assert tuple(out.shape) == (0, 2)
    st = ne.layers.SpatialTransformer()
    out = st([torch.zeros((0, 4, 5, 6, 1), device='cuda'), torch.zeros((0, 4, 5, 6, 3), device='cuda')])
    assert tuple(out.shape) == (0, 4, 5, 6, 1)
    one = torch.randn(1, 1, 1, 1, 1, device='cuda')                     # a single voxel: every sample clamps to it
    out = st([one, torch.full((1, 1, 1, 1, 3), 2.5, device='cuda')])
    assert torch.equal(out, one)
    tiny = ne.utils.resize(torch.randn(4, 4, 4, 1, device='cuda'), 0.2)  # int(4*0.2) = 0 voxels per axis
    assert tuple(tiny.shape) == (0, 0, 0, 1)
    same = torch.randn(2, 3, 4, 5, 1, device='cuda')
    assert ne.layers.Resize(1)(same) is not None and torch.equal(ne.layers.Resize(1)(same), same)   # utils.py:250-251


def test_vxm_adjacent_transforms_vs_oracle(ne):
    """VecInt / ComposeTransform / RescaleTransform (SURVEY 8f item 2) == the same
    compositions of the oracle's warp and resize, bit for bit."""
    rng = np.random.default_rng(41)
    vel = rng.uniform(-4, 4, (2, 12, 16, 32, 3)).astype(F32)
    out = ne.layers.VecInt(int_steps=5)(dev(vel)).cpu().numpy()
    np.testing.assert_array_equal(out, ointerp.vec_int(vel, 5))
    a = rng.uniform(-3, 3, (1, 10, 12, 32, 3)).astype(F32)
    b = rng.uniform(-3, 3, (1, 10, 12, 32, 3)).astype(F32)
    c = rng.uniform(-3, 3, (1, 10, 12, 32, 3)).astype(F32)
    out = ne.layers.ComposeTransform()([dev(a), dev(b), dev(c)]).cpu().numpy()
    np.testing.assert_array_equal(out[0], ointerp.compose([a[0], b[0], c[0]]))
    half = rng.uniform(-2, 2, (2, 6, 8, 10, 3)).astype(F32)
    for z in (2, 0.5):
        out = ne.layers.RescaleTransform(z)(dev(half)).cpu().numpy()
        np.testing.assert_array_equal(out, ointerp.rescale_transform(half, z))


# the last four stage their source (S2·C % 4 == 0) but their voxel pairs cannot leave as 64 / 128-bit stores -- row
# pitch 35, 70 and 105 floats, and an even pitch with an item stride of 90 floats -- so they take the one-voxel staged
# kernel by default
@pytest.mark.parametrize('shape,C,zoom', [((7, 9, 33), 1, 2), ((6, 5, 40), 2, 3), ((5, 6, 35), 3, 2.5), ((4, 7, 34), 4, 4),
                                          ((9, 8, 32), 3, [1.5, 2, 3.7]), ((3, 2, 2), 1, 2), ((10, 12, 70), 3, 1.6),
                                          ((40, 9, 21), 3, [2, 2, 3]), ((5, 33, 17), 2, 2), ((6, 7, 9), 1, [2, 2, 0.6]),
                                          ((33, 18, 20), 4, [0.5, 1.3, 2.1]), ((6, 7, 20), 1, [2, 2, 1.75]),
                                          ((5, 6, 20), 2, [2, 2, 1.75]), ((5, 6, 20), 3, [2, 2, 1.75]),
                                          ((3, 3, 8), 1, [1, 1, 1.25])])
def test_resize_upsampling_vs_oracle(ne, monkeypatch, shape, C, zoom):
    """up-sampling (and mixed) shapes through the TMA-staged tile kernels (voxel-pair kernel: default, even and odd
    output widths, and its global-memory path; one voxel per thread), the one-voxel z-marching kernel (global loads)
    and the generic kernel: -0.0 / rounding identical"""
    rng = np.random.default_rng(51)
    x = rng.standard_normal((2,) + shape + (C,)).astype(F32)
    x[0, 0, 0, :2] = 0.0                                     # exact zeros: the packed a*b = fma(a, b, -0) must keep their sign
    x[1, -1, -1, -3:] = -0.0
    ref = ointerp.resize_layer(x, zoom)
    out = ne.layers.Resize(zoom)(dev(x))
    np.testing.assert_array_equal(out.cpu().numpy(), ref)
    np.testing.assert_array_equal(np.signbit(out.cpu().numpy()), np.signbit(ref))
    monkeypatch.setenv('NRT_RESIZE_UNSTAGED', '1')            # -> pair kernel, every CTA on its global-memory path
    out = ne.layers.Resize(zoom)(dev(x)).cpu().numpy()
    np.testing.assert_array_equal(out, ref)
    np.testing.assert_array_equal(np.signbit(out), np.signbit(ref))
    monkeypatch.delenv('NRT_RESIZE_UNSTAGED')
    monkeypatch.setenv('NRT_RESIZE_TILE_X2', '0')             # -> staged source, one voxel per thread
    np.testing.assert_array_equal(ne.layers.Resize(zoom)(dev(x)).cpu().numpy(), ref)
    monkeypatch.setenv('NRT_RESIZE_TILE', '0')                # -> one-voxel z-marching kernel (global loads)
    np.testing.assert_array_equal(ne.layers.Resize(zoom)(dev(x)).cpu().numpy(), ref)
    monkeypatch.setenv('NRT_RESIZE_GENERIC', '1')
    np.testing.assert_array_equal(ne.layers.Resize(zoom)(dev(x)).cpu().numpy(), ref)


@pytest.mark.parametrize('C', [1, 2, 3, 4])
def test_resize_unaligned_output_vs_oracle(ne, C):
    """nrt_resize_f32 into an output one float past an aligned allocation, from a TMA-able source (S2·C % 4 == 0):
    C = 1, 3 take the one-voxel staged kernel, C = 2, 4 the run-time-C z-marching kernel.  Bit-exact incl. the sign of
    zero, and nothing written outside the output"""
    from neurite_b200._lib import lib, check, ptr, stream_ptr, i32_array, method_id
    rng = np.random.default_rng(52)
    shape, zoom = (5, 6, 20), [2, 2, 1.75]
    x = rng.standard_normal((2,) + shape + (C,)).astype(F32)
    x[0, 0, 0, :2] = 0.0
    x[1, -1, -1, -3:] = -0.0
    ref = ointerp.resize_layer(x, zoom)
    new_shape = ref.shape[1:4]
    buf = torch.full((ref.size + 2,), float('nan'), device='cuda')
    out = buf[1:1 + ref.size]
    assert out.data_ptr() % 16 == 4
    xd = dev(x)
    check(lib.nrt_resize_f32(ptr(xd), ptr(out), 2, i32_array(shape), i32_array(new_shape), 3, C,
                             method_id('linear'), 0, new_shape[0], stream_ptr()))
    got = out.cpu().numpy().reshape(ref.shape)
    np.testing.assert_array_equal(got, ref)
    np.testing.assert_array_equal(np.signbit(got), np.signbit(ref))
    assert torch.isnan(buf[0]) and torch.isnan(buf[-1])


def test_interpn_on_the_volume_grid_uses_tiles_and_stays_exact(ne, monkeypatch):
    """interpn(vol, grid + shift) -- the call voxelmorph's transform() makes -- goes through
    the TMA tile kernel with absolute locations; bit-exact vs the oracle and vs the gather kernel,
    also for locations that have nothing to do with the grid."""
    rng = np.random.default_rng(61)
    S = (20, 24, 64)
    grid = np.stack(np.meshgrid(*[np.arange(s, dtype=F32) for s in S], indexing='ij'), -1)
    for C in (1, 3):
        vol = rng.standard_normal(S + (C,)).astype(F32)
        for loc in ((grid + rng.uniform(-3, 3, grid.shape)).astype(F32),
                    (grid + np.array([7.5, -6.25, 10.0], F32) + rng.uniform(-1, 1, grid.shape)).astype(F32),
                    rng.uniform(-5, 70, grid.shape).astype(F32)):
            for method, fill in (('linear', None), ('nearest', 0.0)):
                ref = ointerp.interpn(vol, loc, method, fill)
                out = ne.utils.interpn(dev(vol), dev(loc), method, fill).cpu().numpy()
                np.testing.assert_array_equal(out, ref)
    monkeypatch.setenv('NRT_WARP_TILE', '0')
    np.testing.assert_array_equal(ne.utils.interpn(dev(vol), dev(loc)).cpu().numpy(), ointerp.interpn(vol, loc))


def test_lc3d_implementations_2_and_3_equal_implementation_1(ne):
    """the layer with the reference's implementation-2 / -3 parameter layouts (converted on the fly) == implementation 1"""
    from neurite_b200 import layers
    rng = np.random.default_rng(77)
    for fmt, xshape in (('channels_last', (3, 6, 5, 7, 4)), ('channels_first', (3, 4, 6, 5, 7))):
        x = dev(rng.standard_normal(xshape).astype(F32))
        l1 = layers.LocallyConnected3D(8, (3, 2, 3), strides=(1, 2, 1), data_format=fmt, activation='relu')
        l1.build(xshape)
        l1 = l1.cuda()
        with torch.no_grad():
            l1.bias.normal_()
            y1 = l1(x)
        for impl in (2, 3):
            li = layers.LocallyConnected3D(8, (3, 2, 3), strides=(1, 2, 1), data_format=fmt, activation='relu', implementation=impl)
            li.build(xshape)
            li = li.cuda()
            with torch.no_grad():
                li.kernel.copy_(layers.lc3d_kernel_to_impl(l1.kernel, impl, l1.input_spatial, l1.input_filter, l1.kernel_size,
                                                           l1.strides, fmt))
                li.bias.copy_(l1.bias)
                assert torch.equal(li(x), y1)
    # gradients reach the implementation-3 weight vector through the re-indexing
    li.kernel.grad = None
    li(x).sum().backward()
    assert li.kernel.grad is not None and tuple(li.kernel.grad.shape) == tuple(li.kernel.shape)


def test_spatial_transformer_single_transform_and_square_affine(ne):
    """ADVICE r1: single_transform applies trf[0] to every volume whatever the transform batch size; affines may come
    as [B, N+1, N+1]; a transform on another grid shares one mesh across the batch."""
    rng = np.random.default_rng(31)
    vol = rng.standard_normal((3, 8, 9, 12, 2)).astype(F32)
    flow = rng.uniform(-2, 2, (3, 8, 9, 12, 3)).astype(F32)
    out = ne.layers.SpatialTransformer(single_transform=True)([dev(vol), dev(flow)]).cpu().numpy()
    ref = ointerp.spatial_transformer(vol, np.repeat(flow[:1], 3, 0))
    np.testing.assert_array_equal(out, ref)
    aff = np.tile(np.eye(4, dtype=F32)[None], (3, 1, 1))
    aff[:, :3, 3] = [[0.5, -1.25, 2.0]] * 3
    aff[:, 0, 1] = 0.03
    a = ne.layers.SpatialTransformer()([dev(vol), dev(aff[:, :3, :])])
    b = ne.layers.SpatialTransformer()([dev(vol), dev(aff)])
    assert torch.equal(a, b)
    small = rng.uniform(-1, 1, (3, 4, 5, 6, 3)).astype(F32)                    # output grid != volume grid
    out = ne.layers.SpatialTransformer()([dev(vol), dev(small)]).cpu().numpy()
    for bi in range(3):
        mesh = np.stack(np.meshgrid(*[np.arange(s, dtype=F32) for s in small.shape[1:-1]], indexing='ij'), -1)
        np.testing.assert_array_equal(out[bi], ointerp.interpn(vol[bi], mesh + small[bi]))
