"""
neurite_b200.augment -- the noise fields of neurite's synthesis generator
(adalca/neurite: neurite/tf/utils/augment.py:65-218), on torch CUDA tensors, channels-last.

    random_blur_rescale(x, std_min, std_max, isotropic, seed, reduce, batched)   augment.py:65-112
    draw_perlin_full(shape, noise_min, noise_max, fwhm_min, fwhm_max, ...)      augment.py:115-218
    draw_crop_mask(x, crop_min, crop_max, axis, prob, bilateral, seed)          augment.py:221-287

Also reachable as `neurite_b200.utils.augment`, as in the reference.

Randomness.  TF's random stream cannot be reproduced outside TF.  The seed chain is the reference's: a numpy
`default_rng(seed)` hands out one integer per draw (per level: SD table, noise, blur), and each blur seed hands out
one integer per spatial axis.  The SD table and the noise are drawn on the device by the Philox4x32-10 stream of
nrt_noise.cu keyed with those integers; the smoothing SDs are drawn on the host from a numpy generator seeded with
them.  So the same seed gives bit-identical output, different draws use independent streams, and torch's global RNG
state is never read or changed.  `seed=None` seeds from the operating system.

The pipeline after the draws (_draw_perlin_full_from_draws) is deterministic: one separable-convolution pass per
item and axis (nrt_sepconv_axis_f32: the taps differ per item), the statistic before and after the blur per item
(nrt_item_stats_f32) and the mean over levels of x * divide_no_nan(before, after) (nrt_level_combine_f32).  The
statistics stay on the device.
"""
import numpy as np
import torch

from . import utils
from ._lib import lib, check, ptr, stream_ptr, i32_array, require_cuda, NRT_STAT_SD, NRT_STAT_MAX

_MAX_SEED = np.iinfo(int).max
_STAT_KIND = {'std': NRT_STAT_SD, 'max': NRT_STAT_MAX}


def normalize_axes(axes, shape, allowed=None, none_means_all=False):
    """Sort, deduplicate and validate axes into [0, N) (neurite/py/utils.py:124-167); IndexError outside
    `allowed`."""
    ndims = len(shape)
    if allowed is None:
        allowed = range(ndims)
    if np.isscalar(allowed):
        allowed = [allowed]
    assert all(ax in range(ndims) for ax in allowed), f'allowed axes {allowed} out of bounds'
    if axes is None:
        axes = allowed if none_means_all else []
    if np.isscalar(axes):
        axes = [axes]
    orig = axes
    axes = [ax + ndims if ax < 0 else ax for ax in axes]
    for ax, inp in zip(axes, orig):
        if ax not in allowed:
            raise IndexError(f'axis {inp} outside {allowed}')
    return tuple(set(axes))


def _seed(rand):
    return int(rand.integers(_MAX_SEED))


def _stat_kind(reduce):
    if callable(reduce):
        return None
    if reduce not in _STAT_KIND:
        raise ValueError(f"reduce must be 'std', 'max' or a callable, got {reduce!r}")
    return _STAT_KIND[reduce]


def _draw_sigmas(rand, std_min, std_max, n_dim, isotropic):
    """random_blur_rescale's kernel SDs (augment.py:102-106 with utils.py:628-653): one draw per axis from
    U[max(std_min, eps), max(std_max, eps)) in fp32; with `isotropic` all draws are consumed and the first is
    used on every axis."""
    f32 = np.float32
    eps = np.finfo(f32).eps
    a, b = f32(max(std_min, eps)), f32(max(std_max, eps))
    sig = []
    for s in rand.integers(_MAX_SEED, size=n_dim):
        s_tf = int(np.random.default_rng(int(s)).integers(_MAX_SEED, size=1)[0])
        u = np.random.default_rng(s_tf).random(dtype=f32)
        sig.append(float(f32(f32(u * f32(b - a)) + a)))
    return sig[:1] * n_dim if isotropic else sig


def _draw_perlin_full_from_draws(noise, sigmas, std_max, reduce='std'):
    """The deterministic rest of draw_perlin_full once the draws are made.

    noise   [L, G, Bg, *space, C] fp32 CUDA tensor: level l of group g, i.e. N(0, sd) as drawn
    sigmas  [L][G][D] smoothing SDs per level, group and spatial axis (isotropic already applied)
    std_max [L] upper SD bound per level: the window is 2 * round(3 * max(std_max, eps)) + 1 taps
    reduce  'std' (population SD), 'max' or a callable applied to each group's [Bg, *space, C] tensor
    -> [G, Bg, *space, C] fp32: mean over levels of blur(x) * divide_no_nan(reduce(x), reduce(blur(x))).
    A group is the tensor one statistic covers: one batch item of PerlinNoise, or the whole batch of
    draw_perlin_full(batched=True)."""
    require_cuda(noise)
    noise = noise.to(torch.float32).contiguous()
    L, G = noise.shape[:2]
    gshape = list(noise.shape[2:])
    D = len(gshape) - 2
    m = int(np.prod(gshape, dtype=np.int64))
    dev = noise.device
    kind = _stat_kind(reduce)

    def stats(t):
        if kind is not None:
            return utils._item_stats(t.reshape(L * G, m), kind)
        return torch.stack([torch.as_tensor(reduce(t[l, g]), device=dev).reshape(())
                            for l in range(L) for g in range(G)]).to(torch.float32)

    before = stats(noise)

    # every tap of every pass in one host buffer, one copy to the device
    eps = np.finfo(np.float32).eps
    taps, offs = [], []
    for l in range(L):
        w = float(np.round(max(std_max[l], eps) * 3) * 2 + 1)
        for g in range(G):
            assert len(sigmas[l][g]) == D, f'{D} SDs expected per group, got {len(sigmas[l][g])}'
            for s in sigmas[l][g]:
                k = utils.gaussian_kernel(sigma=[float(s)], windowsize=[w], separate=True)
                offs.append((sum(t.numel() for t in taps), k.numel()))
                taps.append(k)
    kdev = torch.cat(taps).to(dev) if taps else None

    bufs = (torch.empty_like(noise), torch.empty_like(noise))
    with torch.cuda.device(dev):
        st = stream_ptr(dev)
        for l in range(L):
            for g in range(G):
                src = noise[l, g]
                for a in range(D):
                    dst = bufs[a % 2][l, g]
                    off, K = offs[(l * G + g) * D + a]
                    outer = int(np.prod(gshape[:a + 1], dtype=np.int64))
                    n = gshape[a + 1]
                    inner = int(np.prod(gshape[a + 2:], dtype=np.int64))
                    n_out, pb = utils._same_padding(n, K, 1, 1)
                    check(lib.nrt_sepconv_axis_f32(ptr(src), ptr(dst), outer, n, inner, ptr(kdev[off:off + K]), K,
                                                   1, 1, pb, n_out, st))
                    src = dst
    blurred = bufs[(D - 1) % 2] if D > 0 else noise
    after = stats(blurred)

    out = torch.empty([G] + gshape, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.nrt_level_combine_f32(ptr(blurred), int(L), int(G), m, ptr(before), ptr(after), ptr(out),
                                        stream_ptr(dev)))
    return out


def _level_draws(rand, n_dim, fwhm_min, fwhm_max, isotropic):
    """Per level: (SD-table key, noise key, SDs), consuming the generator in the reference's order."""
    out = []
    for low, upp in zip(fwhm_min, fwhm_max):
        k_sd, k_noise, s_blur = _seed(rand), _seed(rand), _seed(rand)
        sig = _draw_sigmas(np.random.default_rng(s_blur), low / 2.355, upp / 2.355, n_dim, isotropic)
        out.append((k_sd, k_noise, sig))
    return out


def _perlin_noise(group_draws, gshape, shape_sd, noise_min, noise_max, device):
    """The draws of every level and group on the device: SD tables U[noise_min, noise_max] of shape shape_sd and
    noise N(0, SD) of shape gshape -> [L, G, *gshape] fp32."""
    L, G = len(group_draws[0]), len(group_draws)
    n_sd = int(np.prod(shape_sd, dtype=np.int64))
    tables = torch.empty((L, G, max(n_sd, 1)), dtype=torch.float32, device=device)
    noise = torch.empty([L, G] + list(gshape), dtype=torch.float32, device=device)
    sh, shs = i32_array(gshape), i32_array(shape_sd)
    with torch.cuda.device(device):
        st = stream_ptr(device)
        for g, draws in enumerate(group_draws):
            for l, (k_sd, k_noise, _) in enumerate(draws):
                check(lib.nrt_philox_uniform_f32(k_sd, n_sd, float(noise_min), float(noise_max), ptr(tables[l, g]), st))
                check(lib.nrt_philox_normal_f32(k_noise, sh, shs, len(gshape), ptr(tables[l, g]), None, None,
                                                ptr(noise[l, g]), st))
    return noise


def _perlin(group_draws, gshape, shape_sd, noise_min, noise_max, fwhm_max, reduce, device):
    """Draw the SD tables and the noise of every level and group on the device, then the deterministic rest."""
    noise = _perlin_noise(group_draws, gshape, shape_sd, noise_min, noise_max, device)
    sigmas = [[draws[l][2] for draws in group_draws] for l in range(len(fwhm_max))]
    return _draw_perlin_full_from_draws(noise, sigmas, [u / 2.355 for u in fwhm_max], reduce)


def _check_perlin_args(noise_min, noise_max, fwhm_min, fwhm_max):
    assert 0 < noise_min <= noise_max, f'invalid noise-SD bounds {(noise_min, noise_max)}'
    if not hasattr(fwhm_min, '__iter__'):
        fwhm_min = [fwhm_min]
    if not hasattr(fwhm_max, '__iter__'):
        fwhm_max = [fwhm_max]
    assert len(fwhm_min) == len(fwhm_max), 'different number of lower and upper bounds'
    return list(fwhm_min), list(fwhm_max)


def _device(device):
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError('neurite_b200 noise needs a CUDA device (got %s); there is no CPU path' % device)
    return device


def random_blur_rescale(x, std_min=8 / 2.355, std_max=32 / 2.355, isotropic=False, seed=None, reduce='std',
                        batched=False):
    """Smooth the spatial axes of x with a random Gaussian and rescale so that a global statistic of the whole
    tensor (`reduce`: 'std', 'max' or a callable) is unchanged (augment.py:65-112).  x has a trailing feature
    dimension and, with `batched`, a leading batch dimension."""
    require_cuda(x)
    xb = x if batched else x[None]
    n_dim = xb.dim() - 2
    sig = _draw_sigmas(np.random.default_rng(seed), std_min, std_max, n_dim, isotropic)
    out = _draw_perlin_full_from_draws(xb[None, None], [[sig]], [std_max], reduce)[0]
    out = out if batched else out[0]
    return out.to(x.dtype) if x.dtype != torch.float32 else out


def tf_range_f32(width):
    """tf.range(1, delta=1 / width) in fp32 (provenance: contract; TF's RangeOp, restated): delta = 1 / width,
    length ceil(1 / delta) and element i = i * delta, each op rounded once in fp32."""
    f32 = np.float32
    delta = f32(f32(1) / f32(width))
    n = int(np.ceil(f32(f32(1) / delta)))
    return (np.arange(n, dtype=f32) * delta).astype(f32)


def crop_bounds(width, prop_low, prop_cen):
    """The index range [lo, hi) where draw_crop_mask's mask is 1 (augment.py:280-284): prop >= prop_low and
    prop < prop_low + prop_cen in fp32 on prop = tf.range(1, delta=1/width).  prop is non-decreasing, so the mask
    is one contiguous range.  ValueError where the range's length is not `width` (the reference's reshape
    fails there)."""
    f32 = np.float32
    prop = tf_range_f32(width)
    if prop.size != width:
        raise ValueError(f'tf.range(1, delta=1/{width}) has {prop.size} elements, not {width}: cannot reshape the '
                         f'crop mask')
    pl = f32(prop_low)
    ph = f32(pl + f32(prop_cen))
    lo = int(np.searchsorted(prop, pl, side='left'))
    hi = int(np.searchsorted(prop, ph, side='left'))
    return lo, max(lo, hi)


def _draw_crop(shape, crop_min, crop_max, axis, prob, bilateral, seed):
    """draw_crop_mask's draws (augment.py:246-277) on the host -> (axis, lo, hi).  Each of the reference's
    tf.random.uniform calls takes the next integer of a numpy generator seeded with `seed`, and draws from a
    numpy generator seeded with that integer; the fp32 arithmetic on the draws is TF's."""
    f32 = np.float32
    rand = np.random.default_rng(seed)

    def gen():
        return np.random.default_rng(int(rand.integers(_MAX_SEED)))

    axis = normalize_axes(axis, shape, none_means_all=True)
    assert 0 <= crop_min <= crop_max <= 1, f'invalid proportions {crop_min}, {crop_max}'
    prop_cut = f32(crop_max)
    if crop_min < crop_max:
        lo_, hi_ = f32(crop_min), f32(crop_max)
        prop_cut = f32(f32(gen().random(dtype=f32) * f32(hi_ - lo_)) + lo_)
    assert 0 <= prob <= 1, f'{prob} not a probability'
    if prob < 1:
        bit = gen().random(dtype=f32) < f32(prob)
        prop_cut = f32(prop_cut * f32(bit))
    rand_prop = gen().random(dtype=f32)
    if not bilateral:
        rand_prop = f32(rand_prop < f32(0.5))
    prop_low = f32(prop_cut * rand_prop)
    prop_cen = f32(f32(1) - prop_cut)
    ax = axis[int(gen().integers(len(axis)))]
    lo, hi = crop_bounds(int(shape[ax]), prop_low, prop_cen)
    return ax, lo, hi


def draw_crop_mask(x, crop_min=0, crop_max=0.5, axis=None, prob=1, bilateral=False, seed=None):
    """Mask that crops the field of view of x along one axis (augment.py:221-287): 1 on a drawn index range
    [lo, hi) of one drawn axis, 0 elsewhere, with the shape (1, .., width, .., 1) and x's dtype.  A torch
    tensor on x's device for a tensor x, else a numpy array.  The draws are made on the host (_draw_crop)."""
    if isinstance(x, (list, tuple)):
        x = torch.cat(list(x), 0) if torch.is_tensor(x[0]) else np.concatenate(x, 0)
    shape = list(x.shape)
    ax, lo, hi = _draw_crop(shape, crop_min, crop_max, axis, prob, bilateral, seed)
    mshape = [1] * len(shape)
    mshape[ax] = shape[ax]
    mask = np.zeros(shape[ax], np.float32)
    mask[lo:hi] = 1
    mask = mask.reshape(mshape)
    if torch.is_tensor(x):
        return torch.as_tensor(mask, device=x.device).to(x.dtype)
    return mask.astype(np.asarray(x).dtype)


def draw_perlin_full(shape, noise_min=0.01, noise_max=1, fwhm_min=4, fwhm_max=32, isotropic=False, batched=False,
                     featured=False, reduce='std', dtype=torch.float32, axes=None, seed=None, device=None):
    """Perlin-noise tensor of `shape` drawn at full resolution (augment.py:115-218): per level, noise
    N(0, sd) with sd ~ U[noise_min, noise_max] (one SD per index along `axes`), blurred with random FWHMs in
    [fwhm_min, fwhm_max] keeping `reduce` constant, then averaged over levels.  Computed in fp32, cast to
    `dtype` at the end."""
    fwhm_min, fwhm_max = _check_perlin_args(noise_min, noise_max, fwhm_min, fwhm_max)
    device = _device(device)
    rand = np.random.default_rng(seed)
    shape = [int(s) for s in shape]
    axes = normalize_axes(axes, shape, none_means_all=False)
    if not batched:
        shape = [1] + shape
        axes = [ax + 1 for ax in axes]
    if not featured:
        shape = shape + [1]
    shape_sd = [shape[i] if i in axes else 1 for i in range(len(shape))]
    draws = _level_draws(rand, len(shape) - 2, fwhm_min, fwhm_max, isotropic)
    out = _perlin([draws], shape, shape_sd, noise_min, noise_max, fwhm_max, reduce, device)[0]
    if not batched:
        out = out[0]
    if not featured:
        out = out[..., 0]
    return out.to(dtype) if dtype != torch.float32 else out
