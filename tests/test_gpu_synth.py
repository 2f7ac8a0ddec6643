"""GPU tests of the label-to-image generator: every new kernel against oracle/synth.py at ragged sizes, the full
generator given its plan, determinism, no device-to-host copy, and the layer contracts."""
import numpy as np
import pytest
import torch

import neurite_b200 as ne
from neurite_b200._lib import lib, check, ptr, stream_ptr, i32_array
from oracle import synth as osynth, noise as onoise

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
F32 = np.float32


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV)


def _crop_args(shape, crop):
    if crop is None:
        return 1, 1, 0, 1
    ax, lo, hi = crop
    return shape[ax - 1], int(np.prod(shape[ax:], dtype=np.int64)), lo, hi


def _labels(rng, B, shape, nmax):
    return rng.integers(-2, nmax + 3, (B, *shape, 1)).astype(F32) + F32(0.25)        # out-of-range labels too


@pytest.mark.parametrize('M', [1, 3, 4, 17, 32])
@pytest.mark.parametrize('B,shape,crop,use_lut', [(1, (5, 7, 3), None, False), (2, (9, 11), (2, 3, 9), True),
                                                  (3, (4, 5, 7), (1, 1, 3), True)])
def test_label_map_kernels(M, B, shape, crop, use_lut):
    rng = np.random.default_rng(M * 10 + B)
    lab = _labels(rng, B, shape, M + 2)
    V = int(np.prod(shape))
    lut = rng.integers(-1, M + 1, M + 3).astype(np.int32) if use_lut else None
    cl = osynth.crop_labels(lab, crop, shape)
    out = torch.empty(B, *shape, M, device=DEV)
    d_lut = None if lut is None else _t(lut)
    n = 0 if lut is None else lut.size
    d_lab = _t(lab)                                   # every device argument stays referenced until the sync
    check(lib.nrt_label_map_f32(ptr(d_lab), B, V, *_crop_args(shape, crop), ptr(d_lut), n, M, ptr(out),
                                stream_ptr(DEV)))
    assert np.array_equal(out.cpu().numpy(), osynth.label_map(cl, lut, True, M))
    oi = torch.empty(B, *shape, 1, dtype=torch.int32, device=DEV)
    check(lib.nrt_label_map_i32(ptr(d_lab), B, V, *_crop_args(shape, crop), ptr(d_lut), n, ptr(oi),
                                stream_ptr(DEV)))
    assert np.array_equal(oi.cpu().numpy(), osynth.label_map(cl, lut, False, M))


@pytest.mark.parametrize('C', [1, 2, 3])
@pytest.mark.parametrize('B,shape,crop', [(1, (6, 7, 5), None), (2, (13, 9), (1, 2, 11)), (3, (3, 5, 7), (3, 0, 4))])
@pytest.mark.parametrize('with_bias', [False, True])
@pytest.mark.parametrize('nlut', [9, 12280, 13001])          # the LUT in shared memory, at its limit, in global memory
def test_labels_to_image_kernel(C, B, shape, crop, with_bias, nlut):
    rng = np.random.default_rng(C + 7 * B)
    N = 4
    lab = _labels(rng, B, shape, nlut)
    lut = rng.integers(0, N, nlut).astype(np.int32)
    u = rng.random((B, C, N), dtype=F32)
    mn = rng.uniform(0, 0.5, (C, N)).astype(F32)                  # per-channel bounds, [C, N]
    mx = (mn + rng.uniform(0, 1, (C, N))).astype(F32)
    bias = rng.uniform(-0.3, 0.3, (B, *shape, C)).astype(F32) if with_bias else None
    V = int(np.prod(shape))
    img = torch.empty(B, *shape, C, device=DEV)
    mean = torch.empty_like(img) if with_bias else None
    bout = torch.empty_like(img) if with_bias else None
    amax = torch.empty(1, device=DEV)
    nb = lib.nrt_labels_to_image_workspace_bytes()
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    d = [_t(a) for a in (lab, lut, u, mn, mx)] + [None if bias is None else _t(bias)]
    check(lib.nrt_labels_to_image_f32(ptr(d[0]), B, V, C, *_crop_args(shape, crop), ptr(d[1]), nlut, N,
                                      ptr(d[2]), ptr(d[3]), ptr(d[4]), ptr(d[5]),
                                      1, ptr(img), ptr(mean), ptr(bout), ptr(amax), ptr(ws), nb, stream_ptr(DEV)))
    cl = osynth.crop_labels(lab, crop, shape)
    ref_img, ref_mean = osynth.labels_to_image(cl, lut, u, mn, mx, bias)
    got = img.cpu().numpy()
    if with_bias:
        assert np.array_equal(mean.cpu().numpy(), ref_mean)
        np.testing.assert_allclose(bout.cpu().numpy(), np.exp(bias.astype(np.float64)), rtol=4 * 2.0 ** -23)
        # expf within 2 ulp, then one product rounding: 3 * 2^-24 relative
        np.testing.assert_allclose(got, ref_img, rtol=4 * 2.0 ** -23, atol=0)
    else:
        assert np.array_equal(got, ref_img)
    assert float(amax) == float(np.abs(got).max())


@pytest.mark.parametrize('B,shape,C', [(1, (5, 7, 9), 1), (2, (6, 11), 3), (3, (4, 3, 5), 2)])
def test_noise_background_matches_normal_kernel(B, shape, C):
    rng = np.random.default_rng(B)
    x = rng.uniform(0, 2, (B, *shape, C)).astype(F32)
    lab = rng.integers(0, 3, (B, *shape, 1)).astype(F32)
    sd = rng.uniform(0.1, 0.2, (B, C)).astype(F32)
    scale = _t(np.array([1.7], F32))
    bg = np.array([0.1, 0.9, 0.3][:B], F32)
    key = 12345678901
    V = int(np.prod(shape))
    crop = (1, 1, shape[0] - 1)
    out = torch.empty(B, *shape, C, device=DEV)
    d_sd, d_x, d_lab, d_bg = _t(sd), _t(x), _t(lab), _t(bg)
    check(lib.nrt_philox_normal_background_f32(key, B, V, C, ptr(d_sd), ptr(scale), ptr(d_x), ptr(d_lab),
                                               *_crop_args(shape, crop), ptr(d_bg), 0.5, ptr(out),
                                               stream_ptr(DEV)))
    plain = torch.empty_like(out)
    full, sdshape = [B, *shape, C], [B] + [1] * len(shape) + [C]
    check(lib.nrt_philox_normal_f32(key, i32_array(full), i32_array(sdshape), len(full), ptr(d_sd), ptr(scale),
                                    ptr(d_x), ptr(plain), stream_ptr(DEV)))
    cl = osynth.crop_labels(lab, crop, shape)
    clear = (cl[..., 0] == 0) & (bg.reshape((B,) + (1,) * len(shape)) < F32(0.5))
    got, ref = out.cpu().numpy(), plain.cpu().numpy()
    assert np.array_equal(got[~clear], ref[~clear])                        # the same bits as philox_normal_kernel
    assert np.all(got[clear] == 0)
    z = onoise.philox_normal64(key, x.size).reshape(x.shape)
    o = osynth.noise_background(x, z, sd, 1.7, cl, bg, 0.5)
    np.testing.assert_allclose(got, o, rtol=0, atol=4 * onoise.NORMAL_REL * float(np.abs(z).max() * 0.2 * 1.7) + 1e-6)


@pytest.mark.parametrize('B,n,C', [(1, 7, 1), (2, 1023, 3), (3, 40001, 2), (1, 1, 1)])
@pytest.mark.parametrize('gamma', [0.0, 0.5])
def test_item_stats_minmax_then_norm_gamma_kernels(B, n, C, gamma):
    rng = np.random.default_rng(n)
    x = rng.normal(0, 3, (B, n * C)).astype(F32)
    gu = rng.random((B, C), dtype=F32) if gamma else None
    xd = _t(x)
    mnmx = ne.utils._item_stats(xd, ne._lib.NRT_STAT_MINMAX)
    assert np.array_equal(mnmx.cpu().numpy(), np.stack([x.min(1), x.max(1)], 1))
    d_gu = None if gu is None else _t(gu)
    out = ne.utils._norm_gamma(xd, C, mnmx, d_gu, gamma).cpu().numpy()
    ref = osynth.norm_gamma(x.reshape(B, n, C), True, gu, gamma).reshape(B, -1)
    if gamma:
        np.testing.assert_allclose(out, ref, rtol=8 * 2.0 ** -23, atol=1e-7)          # powf within a few ulp
    else:
        assert np.array_equal(out, ref)


def test_minmax_norm_public():
    x = torch.randn(2, 5, 6, 3, device=DEV)
    ref = (x - x.min()) / (x.max() - x.min())
    torch.testing.assert_close(ne.utils.minmax_norm(x), ref, rtol=2e-7, atol=2e-7)
    per = ne.utils.minmax_norm(x, axis=(1, 2, 3))
    xs = x.reshape(2, -1)
    torch.testing.assert_close(per, ((xs - xs.min(1, keepdim=True)[0]) /
                                     (xs.max(1, keepdim=True)[0] - xs.min(1, keepdim=True)[0])).reshape(x.shape),
                               rtol=2e-7, atol=2e-7)
    assert torch.equal(ne.utils.minmax_norm(torch.full((2, 4, 4), 3.0, device=DEV)), torch.zeros(2, 4, 4, device=DEV))
    with pytest.raises(NotImplementedError):
        ne.utils.minmax_norm(x, axis=1)
    with pytest.raises(RuntimeError, match='gradient'):
        ne.utils.minmax_norm(x.clone().requires_grad_())


@pytest.mark.parametrize('dtype', [torch.float32, torch.int32])
def test_random_crop_values_and_gradient(dtype):
    rng = np.random.default_rng(3)
    x = rng.normal(0, 1, (2, 9, 10, 11, 2)).astype(F32)
    xd = _t(x).to(dtype)
    lay = ne.layers.RandomCrop(crop_min=0.2, crop_max=0.6, seed=11)
    lay.build(tuple(xd.shape))
    ax, lo, hi = ne.augment._draw_crop(list(x.shape), 0.2, 0.6, lay.axis, 1, False, 11)
    if dtype == torch.float32:
        xd.requires_grad_()
    y = lay(xd)
    assert np.array_equal(y.detach().cpu().numpy(), osynth.crop_window(xd.detach().cpu().numpy(), ax, lo, hi))
    assert hi - lo < x.shape[ax]
    if dtype == torch.float32:
        g = _t(rng.normal(0, 1, x.shape).astype(F32))
        y.backward(g)
        assert np.array_equal(xd.grad.cpu().numpy(), osynth.crop_window(g.cpu().numpy(), ax, lo, hi))
    assert ne.layers.RandomCrop(prob=0)(xd) is xd


# ---------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------
def _label_input(rng, B, shape, labels):
    return torch.as_tensor(rng.choice(np.asarray(labels), (B, *shape, 1)).astype(np.int32), device=DEV)


CASES = {
    '3d_defaults': dict(labels_in=range(6), in_shape=(16, 18, 20)),
    '2d_dict_subset_int': dict(labels_in={0: 0, 1: 1, 2: 1, 4: 2, 7: 3}, labels_out={1: 1, 4: 2, 7: 2},
                               in_shape=(24, 28), one_hot=False, crop_prob=1, crop_axes=1, zero_background=1,
                               gamma=0, mean_min=[0, 0.2, 0.4, 0.6], mean_max=[0.1, 0.3, 0.5, 1.0], num_chan=2),
    '3d_list_gaps_b2': dict(labels_in=[0, 3, 5, 9], in_shape=(12, 14, 16), out_shape=(10, 12, 14), crop_prob=1,
                            crop_max=0.5, slice_prob=1, normalize=False, noise_max=0, bias_max=0),
    '3d_half_res': dict(labels_in=range(4), in_shape=(16, 16, 20), half_res=True, warp_max=0, blur_max=0,
                        return_mean=True, zero_background=1),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_generator_label_map_and_mean_exact(name):
    kw = dict(CASES[name])
    seeds = {'warp': 1, 'crop': 2, 'mean': 3, 'bias': 4, 'noise': 5, 'background': 6, 'blur': 7, 'slice': 8,
             'gamma': 9}
    seeds = {k: v for k, v in seeds.items() if not ((k == 'warp' and kw.get('warp_max', 2) == 0) or
                                                   (k == 'bias' and kw.get('bias_max', 0.1) == 0) or
                                                   (k == 'background' and kw.get('zero_background', 0) == 0) or
                                                   (k == 'gamma' and kw.get('gamma', 0.5) == 0))}
    gen = ne.models.labels_to_image_new(seeds=seeds, **kw)
    rng = np.random.default_rng(len(name))
    B = 2
    labs = list(kw['labels_in']) + [max(kw['labels_in']) + 2]
    x = _label_input(rng, B, kw['in_shape'], labs)
    plan = gen._draw(x)
    outs = gen._synthesize(x, plan)
    warped, _ = gen.warp_labels(x, plan)
    c = gen.cfg
    shape = [int(s) for s in c['out_shape']]
    cl = osynth.crop_labels(warped.cpu().numpy(), plan['crop'], shape)
    image, lmap = outs[0], outs[1]
    ref_map = osynth.label_map(cl, c['out_lut'], c['one_hot'], c['num_out'])
    assert np.array_equal(lmap.cpu().numpy(), ref_map)
    assert image.shape == (B, *shape, c['num_chan']) and torch.isfinite(image).all()
    if c['normalize']:
        assert float(image.min()) >= 0 and float(image.max()) <= 1
    # the intensities up to the noise, given the plan
    bias = None if plan['bias'] is None else plan['bias'].cpu().numpy()
    ref_img, ref_mean = osynth.labels_to_image(cl, c['gen_lut'], plan['mean_u'].cpu().numpy(), c['mean_min'],
                                               c['mean_max'], bias)
    if c['return_mean']:
        assert np.array_equal(outs[-1].cpu().numpy(), ref_mean)
    # with noise, background, blur and subsample off, the image is the oracle's norm / gamma of the intensities
    if plan['noise'] is None and plan['bg_u'] is None and plan['blur'] is None and plan['slice'] is None:
        gu = None if plan['gamma_u'] is None else plan['gamma_u'].cpu().numpy()
        ref = osynth.norm_gamma(ref_img, c['normalize'], gu, c['gamma'])
        np.testing.assert_allclose(image.cpu().numpy(), ref, rtol=1e-5, atol=1e-6)


def test_generator_noise_stage_against_numpy_philox():
    gen = ne.models.labels_to_image_new(range(5), in_shape=(14, 16, 18), blur_max=0, normalize=False, gamma=0,
                                        bias_max=0, zero_background=1, seeds={'noise': 3, 'mean': 1, 'warp': 2,
                                                                              'background': 4})
    x = _label_input(np.random.default_rng(0), 2, (14, 16, 18), range(5))
    plan = gen._draw(x)
    image = gen._synthesize(x, plan)[0].cpu().numpy()
    warped, _ = gen.warp_labels(x, plan)
    cl = osynth.crop_labels(warped.cpu().numpy(), plan['crop'], [14, 16, 18])
    c = gen.cfg
    img0, _ = osynth.labels_to_image(cl, c['gen_lut'], plan['mean_u'].cpu().numpy(), c['mean_min'], c['mean_max'])
    k_sd, k_noise = plan['noise']
    sd = onoise.philox_uniform(k_sd, 2, c['noise_min'], c['noise_max']).reshape(2, 1)
    z = onoise.philox_normal64(k_noise, img0.size).reshape(img0.shape)
    scale = float(np.abs(img0).max())
    ref = osynth.noise_background(img0, z, sd, scale, cl, plan['bg_u'].cpu().numpy(), 1)
    tol = 2 * onoise.NORMAL_REL * np.abs(z) * c['noise_max'] * scale + 2 ** -22 * (np.abs(ref) + 1)
    assert np.all(np.abs(image - ref) <= tol)


def test_generator_full_size_16_labels():
    gen = ne.models.labels_to_image_new(range(16), in_shape=(160, 192, 224), seeds={'mean': 1, 'warp': 2})
    x = _label_input(np.random.default_rng(1), 1, (160, 192, 224), range(16))
    plan = gen._draw(x)
    image, onehot = gen._synthesize(x, plan)
    warped, _ = gen.warp_labels(x, plan)
    ref = torch.nn.functional.one_hot(warped[..., 0].to(torch.int64), 16).to(torch.float32)
    assert torch.equal(onehot, ref)
    assert float(image.min()) >= 0 and float(image.max()) <= 1


def test_generator_determinism_and_torch_rng_untouched():
    kw = dict(labels_in=range(4), in_shape=(12, 14, 16), crop_prob=1, slice_prob=1, zero_background=0.5)
    seeds = {'warp': 1, 'crop': 2, 'mean': 3, 'bias': 4, 'noise': 5, 'background': 6, 'blur': 7, 'slice': 8,
             'gamma': 9}
    x = _label_input(np.random.default_rng(2), 2, (12, 14, 16), range(4))
    state, cstate = torch.get_rng_state(), torch.cuda.get_rng_state()
    a = ne.models.labels_to_image_new(seeds=seeds, **kw)(x)
    b = ne.models.labels_to_image_new(seeds=seeds, **kw)(x)
    c = ne.models.labels_to_image_new(seeds={k: v + 100 for k, v in seeds.items()}, **kw)(x)
    assert torch.equal(torch.get_rng_state(), state) and torch.equal(torch.cuda.get_rng_state(), cstate)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    assert not torch.equal(a[0], c[0])
    g = ne.models.labels_to_image_new(seeds=seeds, **kw)
    first, second = g(x), g(x)                                  # seed + calls: the second call draws afresh
    assert torch.equal(first[0], a[0]) and not torch.equal(second[0], first[0])


def test_generator_outputs_and_single_output():
    kw = dict(labels_in=range(3), in_shape=(8, 10, 12))
    x = _label_input(np.random.default_rng(3), 2, (8, 10, 12), range(3))
    outs = ne.models.labels_to_image_new(return_vel=True, return_def=True, return_aff=True, return_mean=True,
                                         return_bias=True, **kw)(x)
    assert len(outs) == 7
    assert outs[2].shape == (2, 4, 5, 6, 3) and outs[3].shape == (2, 8, 10, 12, 3)
    assert torch.equal(outs[4], torch.eye(4, device=DEV).expand(2, 4, 4))
    assert outs[5].shape == outs[6].shape == (2, 8, 10, 12, 1) and float(outs[6].min()) > 0
    single = ne.models.labels_to_image_new(return_map=False, **kw)(x)
    assert torch.is_tensor(single) and single.shape == (2, 8, 10, 12, 1)
    fx = ne.models.labels_to_image_new(return_im=False, **kw)(x.to(torch.float32))
    assert fx.shape == (2, 8, 10, 12, 3)


def _kernel_names(fn):
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    if not any(e.device_type == torch.autograd.DeviceType.CUDA for e in prof.events()):
        pytest.skip('torch.profiler recorded no CUDA events on this machine')
    return names


def test_profiler_generator_kernels_and_no_device_to_host_copy():
    gen = ne.models.labels_to_image_new(range(8), in_shape=(16, 16, 16), zero_background=1, seeds={'mean': 1})
    x = _label_input(np.random.default_rng(4), 2, (16, 16, 16), range(8))
    gen(x)
    torch.cuda.synchronize()
    names = _kernel_names(lambda: gen(x))
    for k in ('labels_to_image_kernel', 'absmax_final_kernel', 'philox_normal_background_kernel',
              'item_stats_partial_kernel<false>', 'item_stats_final_kernel<false>', 'norm_gamma_kernel',
              'one_hot_kernel'):
        assert any(k in n for n in names), k
    assert not any('DtoH' in n or 'Device -> Host' in n for n in names), [n for n in names if 'Memcpy' in n]
    gen_i = ne.models.labels_to_image_new(range(8), in_shape=(16, 16, 16), one_hot=False, labels_out={1: 1, 2: 5})
    names = _kernel_names(lambda: gen_i(x))
    assert any('label_map_kernel' in n for n in names) and any('philox_normal_kernel' in n for n in names)
    lay = ne.layers.RandomCrop(seed=1)
    xf = torch.rand(1, 8, 8, 8, 1, device=DEV)
    assert any('crop_window_kernel' in n for n in _kernel_names(lambda: lay(xf)))


# ---------------------------------------------------------------------------------------
# the reference's own generator (tests/golden/synth_*): _synthesize on each fixture's plan
# ---------------------------------------------------------------------------------------
import ast, glob, os  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
SYNTH = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, 'synth_*.npz')))


@pytest.mark.parametrize('name', SYNTH)
def test_synthesize_on_fixture_plan(name):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    kw = ast.literal_eval(str(fx['kwargs']))
    q = [fx['q%d' % i] for i in range(int(fx['nq']))]
    labels = fx['labels']
    c, p = osynth.decode_synth(kw, labels, q)
    gen = ne.models.labels_to_image_new(**dict(kw, return_mean=True, return_vel=False, return_def=False,
                                                 return_bias=False))
    plan = {
        'vel': None if p['vel'] is None else _t(p['vel']),
        'crop': p['crop'],
        'mean_u': _t(p['mean_u']),
        'bias': None if p['bias'] is None else _t(p['bias']),
        'noise': None if p['noise'] is None else (11, 12),
        'bg_u': None if p['bg_u'] is None else _t(p['bg_u']),
        'blur': None if p['blur'] is None else ([float(s) for s in p['blur'][0]], p['blur'][1]),
        'slice': None if p['slice'] is None else (p['slice'][0], ne.utils.subsample_indices(
            c['out_shape_eff'][p['slice'][0] - 1], p['slice'][1])),
        'gamma_u': None if p['gamma_u'] is None else _t(p['gamma_u']),
    }
    outs = gen._synthesize(_t(labels), plan)
    image, lmap, mean = outs[0], outs[1], outs[-1]
    if p['noise'] is not None:                  # the device draws Philox normals for keys (11, 12): the same z here
        u_sd = onoise.philox_uniform(11, p['mean_u'].shape[0] * c['num_chan'], 0, 1)
        p = dict(p, noise=(u_sd.reshape(-1, c['num_chan']), None))
    z = None
    if p['noise'] is not None:
        n = labels.shape[0] * int(np.prod(c['out_shape_eff'])) * c['num_chan']
        z = onoise.philox_normal64(12, n).reshape([labels.shape[0]] + c['out_shape_eff'] + [c['num_chan']])
    r = osynth.synth_from_plan(labels, c, p, z=z)
    ref_outs = [fx['out%d' % i] for i in range(int(fx['nout']))]
    assert np.array_equal(lmap.cpu().numpy(), ref_outs[1])                    # the reference's own label map
    assert np.array_equal(mean.cpu().numpy(), r['mean'])                     # bit-exact uncorrupted mean
    if kw.get('return_mean'):
        assert np.array_equal(r['mean'], ref_outs[len(ref_outs) - 1 - int(bool(kw.get('return_bias')))])
    lo, hi = osynth.image_interval(r, c, p, z)
    got = image.cpu().numpy().astype(np.float64)
    assert np.all((got >= lo) & (got <= hi)), float(np.max(np.maximum(lo - got, got - hi)))
    if p['noise'] is None:
        # without noise the plan is the fixture's own: the image is the reference's within the same interval
        ref_im = ref_outs[0].astype(np.float64)
        assert np.all((ref_im >= lo) & (ref_im <= hi))
