"""
GPU tests of PerlinNoise / GaussianNoise / draw_perlin_full / random_blur_rescale (nrt_noise.cu and the blur
passes of nrt_conv.cu): the golden fixtures through _draw_perlin_full_from_draws against the fp64 graph of
oracle/noise.py, the Philox stream against its numpy restatement, distribution checks on fixed seeds, the
per-item statistics, determinism, the layer contracts.

Bound: |got - ref| <= 4 k 2^-24 scale (oracle/noise.perlin_bounds: k and scale from the blur passes' taps, the
statistics and the level mean).
"""
import re

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import noise as onoise

pytestmark = pytest.mark.gpu
F32 = np.float32
U = 2.0 ** -24


@pytest.fixture(scope='module')
def ne(cuda):
    import neurite_b200
    return neurite_b200


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def check_perlin(ne, d):
    got = ne.augment._draw_perlin_full_from_draws(dev(d['noise']), d['sigmas'], d['std_max'], d['reduce'])
    ref, parts = onoise.torch_perlin64(d['noise'], d['sigmas'], d['std_max'], d['reduce'])
    scale, k = onoise.perlin_bounds(parts, d['reduce'])
    err = (got.cpu().double() - ref).abs()
    tol = 4 * k * U * scale
    assert bool((err <= tol).all()), 'max err/tol %.3g' % float((err / tol.clamp_min(1e-300)).max())
    return got


# ------------------------------------------------------------------ the pipeline given the draws
@pytest.mark.parametrize('name', golden_names('perlin_'))
def test_golden_from_draws(ne, name):
    d = onoise.decode_perlin(load_golden(name))
    got = check_perlin(ne, d)
    assert got.shape == d['out'].shape


@pytest.mark.parametrize('reduce', ['std', 'max'])
def test_165_tap_blur_passes(ne, reduce):
    """FWHM 64 (sigma 27.2): 165 taps per axis, the bias-field width at 160x192x224.  Axes 0 and 1 of a
    single-channel volume run sepconv_col_kernel, the last axis sepconv_row_kernel."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, 1, 1, 40, 36, 180, 1)).astype(F32)
    sm = 64 / 2.355
    assert onoise.window(sm) == 165
    sig = [[[27.0, 25.5, 20.25]], [[27.1, 26.0, 24.0]]]
    check_perlin(ne, dict(noise=x, sigmas=sig, std_max=[sm, sm], reduce=reduce))


def test_callable_reduce(ne):
    rng = np.random.default_rng(6)
    x = rng.standard_normal((1, 2, 1, 12, 14, 2)).astype(F32)
    sig = [[[1.5, 2.0], [0.7, 1.1]]]
    a = ne.augment._draw_perlin_full_from_draws(dev(x), sig, [2.5], 'std')
    b = ne.augment._draw_perlin_full_from_draws(dev(x), sig, [2.5], lambda t: t.std(unbiased=False))
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------ the generator
def test_uniform_bit_exact(ne):
    n, key = 100003, 0x123456789abcdef
    out = torch.empty(n, device='cuda')
    ne._lib.check(ne._lib.lib.nrt_philox_uniform_f32(key, n, 0.25, 3.5, ne._lib.ptr(out), ne._lib.stream_ptr()))
    np.testing.assert_array_equal(out.cpu().numpy(), onoise.philox_uniform(key, n, 0.25, 3.5))


def normal(ne, key, shape, sd, sd_shape, x=None, scale=None):
    out = torch.empty(shape, device='cuda')
    L = ne._lib
    L.check(L.lib.nrt_philox_normal_f32(key, L.i32_array(shape), L.i32_array(sd_shape), len(shape), L.ptr(sd),
                                        L.ptr(scale), L.ptr(x), L.ptr(out), L.stream_ptr()))
    return out


@pytest.mark.parametrize('shape,sd_shape', [((1001,), (1,)), ((2, 5, 7, 3), (2, 1, 1, 3)),
                                            ((3, 4, 5, 6, 7), (1, 4, 1, 6, 1)), ((6, 9, 2), (6, 9, 2))])
def test_normal_within_documented_bound(ne, shape, sd_shape):
    key = 987654321
    n_sd = int(np.prod(sd_shape))
    sd = onoise.philox_uniform(11, n_sd, 0.5, 2.0)
    got = normal(ne, key, list(shape), dev(sd), list(sd_shape)).cpu().numpy().astype(np.float64)
    n = int(np.prod(shape))
    ref = onoise.philox_normal64(key, n).reshape(shape) * np.broadcast_to(sd.reshape(sd_shape), shape)
    assert np.all(np.abs(got - ref) <= (onoise.NORMAL_REL + 2 * U) * np.abs(ref))


def test_geometry_independence(ne):
    n = 4099
    sd = dev(np.ones(1, F32))
    a = normal(ne, 77, [n], sd, [1]).cpu()
    b = normal(ne, 77, [n + 5], sd, [1]).cpu()
    assert torch.equal(a, b[:n])
    ua, ub = torch.empty(n, device='cuda'), torch.empty(n + 5, device='cuda')
    for t in (ua, ub):
        ne._lib.check(ne._lib.lib.nrt_philox_uniform_f32(77, t.numel(), 0.0, 1.0, ne._lib.ptr(t), ne._lib.stream_ptr()))
    assert torch.equal(ua.cpu(), ub.cpu()[:n])


def test_distribution(ne):
    from scipy import stats
    n = 1 << 24
    sds = np.array([0.5, 2.0], F32)
    out = normal(ne, 2024, [n // 2, 2], dev(sds), [1, 2]).cpu().numpy().astype(np.float64)
    for c in range(2):
        z = out[:, c] / sds[c]
        assert abs(z.mean()) < 5 / np.sqrt(z.size)
        assert abs(out[:, c].var() / sds[c] ** 2 - 1) < 5 * np.sqrt(2 / z.size)
        assert stats.kstest(z, 'norm').pvalue > 1e-4
    flat = out.reshape(-1) / np.tile(sds, n // 2)
    assert abs(np.corrcoef(flat[:-1], flat[1:])[0, 1]) < 5 / np.sqrt(n)                  # lag 1
    assert abs(np.corrcoef(out[:, 0], out[:, 1])[0, 1]) < 5 / np.sqrt(n / 2)              # channels
    u = torch.empty(n, device='cuda')
    ne._lib.check(ne._lib.lib.nrt_philox_uniform_f32(5, n, 0.0, 1.0, ne._lib.ptr(u), ne._lib.stream_ptr()))
    assert stats.kstest(u.cpu().numpy(), 'uniform').pvalue > 1e-4


def test_items_and_levels_are_independent(ne):
    """The keys PerlinNoise derives for two items and two levels give uncorrelated noise."""
    lay = ne.layers.PerlinNoise(fwhm_min=[2, 3], fwhm_max=[4, 6], seed=1)
    x = torch.zeros(2, 64, 64, 32, 1, device='cuda')
    lay.build(tuple(x.shape))
    draws, gshape, shape_sd = lay._plan(x, 1)
    noise = ne.augment._perlin_noise(draws, gshape, shape_sd, 1.0, 1.0, x.device).reshape(4, -1).cpu().numpy()
    c = np.corrcoef(noise)
    m = noise.shape[1]
    assert np.all(np.abs(c[~np.eye(4, dtype=bool)]) < 5 / np.sqrt(m))


# ------------------------------------------------------------------ statistics
def test_item_stats_every_kind_against_numpy_and_fp64(ne):
    """Every kind of nrt_item_stats_f32: odd n with several items (rows alternate between float4 and scalar
    loads), n = 1, a base one float past an aligned allocation, and one item large enough to reach the grid cap."""
    L = ne._lib
    stats = ne.utils._item_stats
    rng = np.random.default_rng(3)
    for items, n, offset in ((3, 100001, 0), (1, 7, 0), (5, 4097, 0), (4, 1, 0), (3, 1027, 1), (1, 5000003, 0)):
        x = (rng.standard_normal((items, n)) * 3 + 5).astype(F32)
        buf = torch.empty(items * n + offset, device='cuda')
        xd = buf[offset:].view(items, n)
        xd.copy_(torch.from_numpy(x))
        sd = stats(xd, L.NRT_STAT_SD).cpu().numpy()
        np.testing.assert_allclose(sd, x.astype(np.float64).std(1), rtol=2 * U, atol=0)
        assert np.array_equal(stats(xd, L.NRT_STAT_MAX).cpu().numpy(), x.max(1))
        assert np.array_equal(stats(xd, L.NRT_STAT_ABSMAX).cpu().numpy(), np.abs(x).max(1))
        assert np.array_equal(stats(xd, L.NRT_STAT_MINMAX).cpu().numpy(), np.stack([x.min(1), x.max(1)], 1))
        if offset:                                   # the summation order does not depend on the address
            assert np.array_equal(stats(dev(x), L.NRT_STAT_SD).cpu().numpy(), sd)
    c = dev(np.full((2, 12345), 0.1, F32))
    assert torch.equal(stats(c, L.NRT_STAT_SD).cpu(), torch.zeros(2))


def test_constant_input_gives_zero(ne):
    """std of a constant item is 0, so divide_no_nan makes the rescaled field 0."""
    x = np.full((1, 1, 1, 9, 10, 1), 0.3, F32)
    out = ne.augment._draw_perlin_full_from_draws(dev(x), [[[1.0, 1.5]]], [2.0], 'std')
    assert torch.equal(out.cpu(), torch.zeros_like(out.cpu()))


# ------------------------------------------------------------------ layers
def test_perlin_layer_matches_oracle_given_its_draws(ne):
    lay = ne.layers.PerlinNoise(shape=(14, 15, 16, 3), fwhm_min=[2, 4], fwhm_max=[4, 8], axes=-1, reduce='max', seed=9)
    x = torch.zeros(2, 1, 1, 1, 1, device='cuda')             # rank 5: axes=-1 is the feature axis
    out = lay(x)
    draws, gshape, shape_sd = lay._plan(x, 9)
    noise = ne.augment._perlin_noise(draws, gshape, shape_sd, lay.noise_min, lay.noise_max, x.device)
    sig = [[draws[g][l][2] for g in range(2)] for l in range(2)]
    d = dict(noise=noise.cpu().numpy(), sigmas=sig, std_max=[4 / 2.355, 8 / 2.355], reduce='max')
    ref = onoise.perlin_from_draws(d['noise'], d['sigmas'], d['std_max'], 'max')
    assert out.shape == (2, 14, 15, 16, 3)
    r64, parts = onoise.torch_perlin64(**d)
    scale, k = onoise.perlin_bounds(parts, 'max')
    assert bool(((out.cpu().double() - r64.reshape(out.shape)).abs() <= 4 * k * U * scale.reshape(out.shape)).all())
    np.testing.assert_allclose(out.cpu().numpy(), ref.reshape(out.shape), rtol=1e-4, atol=1e-6)


def test_same_seed_identical_different_seed_differs(ne):
    x = torch.zeros(2, 20, 21, 22, 2, device='cuda')
    a = ne.layers.PerlinNoise(fwhm_min=2, fwhm_max=6, seed=4)(x)
    b = ne.layers.PerlinNoise(fwhm_min=2, fwhm_max=6, seed=4)(x)
    c = ne.layers.PerlinNoise(fwhm_min=2, fwhm_max=6, seed=5)(x)
    assert torch.equal(a, b) and not torch.equal(a, c)
    assert not torch.equal(a[0], a[1])                                # fresh draws per item
    lay = ne.layers.PerlinNoise(fwhm_min=2, fwhm_max=6, seed=4)
    assert torch.equal(lay(x), a) and not torch.equal(lay(x), a)      # seed + calls
    xg = torch.randn(2, 10, 11, 12, 1, device='cuda')
    g1 = ne.layers.GaussianNoise(seed=3)(xg)
    g2 = ne.layers.GaussianNoise(seed=3)(xg)
    g3 = ne.layers.GaussianNoise(seed=4)(xg)
    assert torch.equal(g1, g2) and not torch.equal(g1, g3)
    f = ne.utils.augment.draw_perlin_full((12, 13, 14), fwhm_min=[2, 3], fwhm_max=[4, 5], seed=8)
    assert f.shape == (12, 13, 14) and torch.equal(f, ne.augment.draw_perlin_full((12, 13, 14), fwhm_min=[2, 3],
                                                                                  fwhm_max=[4, 5], seed=8))


def test_rng_state_untouched(ne):
    s_cuda, s_cpu = torch.cuda.get_rng_state(), torch.get_rng_state()
    x = torch.ones(1, 16, 16, 16, 1, device='cuda')
    ne.layers.PerlinNoise(fwhm_min=2, fwhm_max=4)(x)
    ne.layers.GaussianNoise()(x)
    ne.utils.augment.random_blur_rescale(x[0], std_min=0.5, std_max=1.5)
    assert torch.equal(torch.cuda.get_rng_state(), s_cuda) and torch.equal(torch.get_rng_state(), s_cpu)


def test_profiler_no_device_to_host_copy(ne):
    from torch.profiler import profile, ProfilerActivity
    x = torch.randn(2, 24, 28, 32, 1, device='cuda')
    per = ne.layers.PerlinNoise(fwhm_min=[2, 4], fwhm_max=[4, 8], reduce='std', seed=0)
    gau = ne.layers.GaussianNoise(seed=0)
    per(x), gau(x)
    torch.cuda.synchronize()

    # one profiling session for both calls: a second session in the same process may report no CUDA kernels
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        per(x)
        gau(x)
        torch.cuda.synchronize()
    names = [re.sub(r'\s+', '', e.name) for e in prof.events()]
    if not any('kernel' in n for n in names):
        pytest.skip('torch.profiler recorded no CUDA kernels on this machine')
    assert not any('DtoH' in n or 'DeviceToHost' in n for n in names), [n for n in names if 'DtoH' in n]
    # PerlinNoise: the draws, the blur passes, the SDs and the level mean; GaussianNoise: the SD table, max|x| and
    # the fused x + noise pass (philox_uniform / philox_normal / item_stats_*<true> for SD, <false> for max|x|)
    for k in ('philox_uniform_kernel', 'philox_normal_kernel', 'item_stats_partial_kernel<true>',
              'item_stats_final_kernel<true>', 'item_stats_partial_kernel<false>', 'item_stats_final_kernel<false>',
              'level_combine_kernel', 'sepconv_'):
        assert any(k in n for n in names), k


def test_gaussian_noise_only_plus_x_is_full(ne):
    x = torch.randn(2, 9, 10, 11, 3, device='cuda')
    for absolute in (False, True):
        full = ne.layers.GaussianNoise(seed=12, absolute=absolute)(x)
        only = ne.layers.GaussianNoise(seed=12, absolute=absolute, noise_only=True)(x)
        assert torch.equal(only + x, full)


@pytest.mark.parametrize('absolute', [False, True])
def test_gaussian_sd_scaling(ne, absolute):
    x = torch.randn(2, 9, 10, 11, 3, device='cuda') * 4
    lay = ne.layers.GaussianNoise(noise_min=0.1, noise_max=0.2, noise_only=True, absolute=absolute, seed=21)
    got = lay(x).cpu().numpy().astype(np.float64)
    rand = np.random.default_rng(21)
    k_sd, k_noise = int(rand.integers(np.iinfo(int).max)), int(rand.integers(np.iinfo(int).max))
    sd = onoise.philox_uniform(k_sd, 6, 0.1, 0.2).reshape(2, 1, 1, 1, 3).astype(np.float64)
    if not absolute:
        sd = sd * float(x.abs().max())
    ref = onoise.philox_normal64(k_noise, x.numel()).reshape(x.shape) * sd
    assert np.all(np.abs(got - ref) <= (onoise.NORMAL_REL + 3 * U) * np.abs(ref))


def test_gaussian_gradients(ne):
    x = torch.randn(1, 6, 7, 8, 1, device='cuda', requires_grad=True)
    y = ne.layers.GaussianNoise(absolute=True, seed=0)(x)
    y.sum().backward()
    assert torch.equal(x.grad, torch.ones_like(x))
    with pytest.raises(RuntimeError, match='max'):
        ne.layers.GaussianNoise(seed=0)(x)


def test_config_round_trip_and_exceptions(ne):
    P, G = ne.layers.PerlinNoise, ne.layers.GaussianNoise
    p = P(shape=(8, 8, 1), noise_min=0.1, noise_max=0.5, fwhm_min=[2, 3], fwhm_max=[4, 5], isotropic=True,
          reduce='max', axes=-1, seed=3)
    cfg = p.get_config()
    assert set(cfg) >= {'shape', 'noise_min', 'noise_max', 'fwhm_min', 'fwhm_max', 'isotropic', 'reduce',
                        'out_type', 'axes', 'seed'}
    assert P.from_config(cfg).get_config() == cfg
    g = G(noise_min=0.2, noise_max=0.3, noise_only=True, absolute=True, axes=(0, 1), seed=2)
    assert G.from_config(g.get_config()).get_config() == g.get_config()
    x = torch.zeros(1, 8, 8, 1, device='cuda')
    with pytest.raises(IndexError):
        P(axes=0)(x)
    with pytest.raises(AssertionError):
        P(noise_min=0.5, noise_max=0.1)(x)
    with pytest.raises(AssertionError):
        P(fwhm_min=[1, 2], fwhm_max=[3])(x)
    with pytest.raises(AssertionError):
        G(axes=7)(x)
    with pytest.raises(NotImplementedError):
        G()(torch.zeros(1, 4, 4, 1, dtype=torch.complex64, device='cuda'))
    assert G(noise_max=0)(x) is x
    assert P(out_type=torch.float16, seed=1)(x).dtype == torch.float16
