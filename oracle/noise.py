"""
The noise fields of the synthesis generator.  TEST INFRASTRUCTURE (see oracle/__init__.py).

    philox4x32_10 / philox_uniform / philox_normal64   numpy restatement of the Philox4x32-10 stream of
                                                       neurite_b200/csrc/nrt_noise.cu and its normal transform
    sigma_from_draw, perlin_from_draws                 neurite/tf/utils/augment.py:65-218 in numpy fp32, one
                                                       rounding per TF op, given the raw draws
    gaussian_noise_from_draws                          neurite/tf/layers.py:2368-2403 given the raw draws
    decode_perlin / decode_gaussian                    the replayed draw queue of a tests/golden/{perlin,gaussnoise}_*
                                                       fixture -> the draws
    torch_perlin64, perlin_bounds                      the same graph in float64 on the fp32 draws, and the
                                                       per-element bound |got - ref| <= 4 k 2^-24 scale of
                                                       oracle/forward.py for a fp32 evaluation of it

A raw draw is what TF's random ops start from: U[0, 1) for uniform, N(0, 1) for normal.  TF's fp32 arithmetic
on top of them is restated: uniform `u * (maxval - minval) + minval`, normal `z * stddev`.
"""
import numpy as np
import torch

from . import conv
from .forward import torch_separable_conv

F32 = np.float32
EPS32 = float(np.finfo(F32).eps)

# |z - z_exact| <= NORMAL_REL * |z| for the device's Box-Muller normal (nrt_noise.cu): logf 1 ulp halved by
# the root, the root's rounding, sincospif 1 ulp and the product's rounding: 2.5 * 2^-23, rounded up.
NORMAL_REL = 3 * 2.0 ** -23

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


# ---------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------
def philox4x32_10(key, blocks):
    """The four 32-bit words of Philox4x32-10 with key {key & 0xffffffff, key >> 32} and counter
    {j & 0xffffffff, j >> 32, 0, 0} for every j in `blocks`: uint32 [len(blocks), 4]."""
    key = int(key)
    j = np.asarray(blocks, dtype=np.uint64)
    x0, x1 = j & _LO, j >> np.uint64(32)
    x2, x3 = np.zeros_like(j), np.zeros_like(j)
    k0, k1 = key & 0xFFFFFFFF, (key >> 32) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * x0, _M1 * x2
        hi0, lo0 = p0 >> np.uint64(32), p0 & _LO
        hi1, lo1 = p1 >> np.uint64(32), p1 & _LO
        x0, x1, x2, x3 = hi1 ^ x1 ^ np.uint64(k0), lo1, hi0 ^ x3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return np.stack([x0, x1, x2, x3], -1).astype(np.uint32)


def philox_words(key, n):
    """word i % 4 of block i // 4, for i < n."""
    return philox4x32_10(key, np.arange(-(-n // 4))).reshape(-1)[:n]


def u01(w):
    """((w >> 8) + 1) * 2^-24: exact in fp32, in (0, 1]."""
    return ((np.asarray(w, np.uint32) >> np.uint32(8)) + np.uint32(1)).astype(F32) * F32(2.0 ** -24)


def philox_uniform(key, n, lo, hi):
    """nrt_philox_uniform_f32: lo + (hi - lo) * u in fp32, each op rounded once (bit-exact to the device)."""
    lo, hi = F32(lo), F32(hi)
    return (u01(philox_words(key, n)) * F32(hi - lo) + lo).astype(F32)


def philox_normal64(key, n):
    """The standard normals of nrt_philox_normal_f32 evaluated in float64 on the same uniforms: pairs of words
    (w0, w1), (w2, w3) of each block give r = sqrt(-2 log u_even), z_even = r cos(2 pi u_odd),
    z_odd = r sin(2 pi u_odd)."""
    nb = -(-n // 4)
    u = u01(philox4x32_10(key, np.arange(nb))).astype(np.float64)
    r = np.sqrt(-2.0 * np.log(u[:, 0::2]))
    th = 2.0 * np.pi * u[:, 1::2]
    z = np.empty((nb, 4), np.float64)
    z[:, 0::2] = r * np.cos(th)
    z[:, 1::2] = r * np.sin(th)
    return z.reshape(-1)[:n]


# ---------------------------------------------------------------------------------------
# the pipeline given the draws, fp32
# ---------------------------------------------------------------------------------------
def uniform_from_draw(u, lo, hi):
    """tf.random.uniform on a raw U[0, 1) draw: u * (hi - lo) + lo in fp32."""
    lo, hi = F32(lo), F32(hi)
    return (np.asarray(u, F32) * F32(hi - lo) + lo).astype(F32)


def sigma_from_draw(u, std_min, std_max):
    """gaussian_kernel(random=True)'s SD (utils.py:628-653): U[max(std_min, eps), max(std_max, eps)) in fp32."""
    return uniform_from_draw(u, max(std_min, EPS32), max(std_max, EPS32)).reshape(())


def window(std_max):
    return float(np.round(max(std_max, EPS32) * 3) * 2 + 1)


def blur_kernels(sigmas, std_max):
    return [np.asarray(conv.gaussian_kernel([float(s)], windowsize=[window(std_max)], separate=True), F32)
            for s in sigmas]


def _reduce(x, reduce):
    if reduce == 'std':
        return F32(np.std(x.astype(np.float64)))       # population SD, float64 then one rounding
    return F32(np.max(x))


def _divide_no_nan(a, b):
    return F32(0) if b == 0 else F32(F32(a) / F32(b))


def perlin_from_draws(noise, sigmas, std_max, reduce='std'):
    """augment.py:101-113 + 212-213 per group: noise [L, G, Bg, *space, C] fp32, sigmas [L][G][D], std_max [L]
    -> [G, Bg, *space, C]: mean over levels of blur(x) * divide_no_nan(reduce(x), reduce(blur(x)))."""
    noise = np.asarray(noise, F32)
    L, G = noise.shape[:2]
    out = np.zeros(noise.shape[1:], F32)
    for g in range(G):
        lev = []
        for l in range(L):
            x = noise[l, g]
            y = conv.separable_conv(x, blur_kernels(sigmas[l][g], std_max[l]), batched=True)
            lev.append((y * _divide_no_nan(_reduce(x, reduce), _reduce(y, reduce))).astype(F32))
        out[g] = np.mean(np.stack(lev), axis=0, dtype=np.float64).astype(F32)
    return out


def gaussian_noise_from_draws(x, u_sd, z, noise_min, noise_max, noise_only=False, absolute=False):
    """GaussianNoise.call (layers.py:2368-2403) on raw draws: sd = uniform(u_sd) [* max|x|], out = [x +] z * sd."""
    x = np.asarray(x, F32)
    sd = uniform_from_draw(u_sd, noise_min, noise_max)
    if not absolute:
        sd = (sd * np.max(np.abs(x))).astype(F32)
    noise = (np.asarray(z, F32) * sd).astype(F32)
    return noise if noise_only else (x + noise).astype(F32)


# ---------------------------------------------------------------------------------------
# the fixtures' draw queues
# ---------------------------------------------------------------------------------------
def _queue(fx):
    return [fx['q%d' % i] for i in range(int(fx['nq']))]


def decode_perlin(fx):
    """A perlin_* fixture (perlin_blur_rescale_*: random_blur_rescale) -> dict(noise [L, G, Bg, *space, C], sigmas [L][G][D],
    std_max [L], reduce, isotropic, out [G, Bg, *space, C], levels [L][G] (u_sd, z, u_sigmas))."""
    q = _queue(fx)
    reduce = str(fx['reduce'])
    iso = bool(fx['isotropic'])
    if 'std_min' in fx.files:                        # random_blur_rescale(x, batched=True): one group, one level
        x = np.asarray(fx['x'], F32)
        D = x.ndim - 2
        sig = [sigma_from_draw(u, float(fx['std_min']), float(fx['std_max'])) for u in q[:D]]
        sig = sig[:1] * D if iso else sig
        return dict(noise=x[None, None], sigmas=[[sig]], std_max=[float(fx['std_max'])], reduce=reduce,
                    out=np.asarray(fx['out'], F32)[None], isotropic=iso)
    fmin, fmax = [float(v) for v in np.ravel(fx['fwhm_min'])], [float(v) for v in np.ravel(fx['fwhm_max'])]
    nmin, nmax = float(fx['noise_min']), float(fx['noise_max'])
    if 'x' in fx.files:                              # PerlinNoise: one group per batch item, gshape [1, *shape]
        x = fx['x']
        shape = list(fx['shape']) if 'shape' in fx.files else list(x.shape[1:])
        G, gshape = x.shape[0], [1] + [int(s) for s in shape]
    else:                                            # draw_perlin_full
        shape = [int(s) for s in fx['shape']]
        gshape = ([] if bool(fx['batched']) else [1]) + shape + ([] if bool(fx['featured']) else [1])
        G = 1
    L, D = len(fmin), len(gshape) - 2
    noise = np.zeros([L, G] + gshape, F32)
    sigmas = [[None] * G for _ in range(L)]
    k = 0
    for g in range(G):
        for l in range(L):
            u_sd, z, us = q[k], q[k + 1], q[k + 2:k + 2 + D]
            k += 2 + D
            sd = uniform_from_draw(u_sd, nmin, nmax)
            noise[l, g] = (np.asarray(z, F32) * sd).astype(F32)
            sig = [sigma_from_draw(u, fmin[l] / 2.355, fmax[l] / 2.355) for u in us]
            sigmas[l][g] = sig[:1] * D if iso else sig
    assert k == len(q), 'draw queue not consumed: %d of %d' % (k, len(q))
    return dict(noise=noise, sigmas=sigmas, std_max=[f / 2.355 for f in fmax], reduce=reduce, isotropic=iso,
                out=np.asarray(fx['out'], F32).reshape([G] + gshape))


def decode_gaussian(fx):
    q = _queue(fx)
    kw = {k: fx[k].item() for k in ('noise_min', 'noise_max', 'noise_only', 'absolute') if k in fx.files}
    return q[0], q[1], kw


# ---------------------------------------------------------------------------------------
# float64 graph and bound
# ---------------------------------------------------------------------------------------
def torch_perlin64(noise, sigmas, std_max, reduce='std'):
    """perlin_from_draws in float64 on the fp32 draws and fp32 kernels.  Returns (out [G, ...], parts) with
    parts[l][g] = (blur64, ratio64, scale_blur, K total): what perlin_bounds needs."""
    noise = torch.as_tensor(np.asarray(noise, F32)).double()
    L, G = noise.shape[:2]
    D = noise.dim() - 4
    out = torch.zeros(noise.shape[1:], dtype=torch.float64)
    parts = [[None] * G for _ in range(L)]
    red = (lambda t: t.std(unbiased=False)) if reduce == 'std' else (lambda t: t.max())
    for l in range(L):
        for g in range(G):
            ks = blur_kernels(sigmas[l][g], std_max[l])
            x = noise[l, g]
            y = torch_separable_conv(x, ks, list(range(D)))
            sb = torch_separable_conv(x.abs(), [np.abs(k) for k in ks], list(range(D)))
            b, a = red(x), red(y)
            r = b / a if float(a) != 0 else torch.zeros((), dtype=torch.float64)
            out[g] += y * r / L
            parts[l][g] = (y, r, sb, sum(k.size for k in ks))
    return out, parts


def perlin_bounds(parts, reduce='std'):
    """(scale, k) of every output element of the fp32 pipeline against torch_perlin64:
      blur          the D passes: depth sum K + D on scale_blur = |k| * |x| (forward.sepconv_bounds);
      statistic     a blur error moves reduce(blur) by at most rms(scale_blur) (std) or max(scale_blur) (max):
                    relative to reduce(blur) it reaches the element as |blur| * that / |reduce(blur)|;
      the rest      reduce(x) and reduce(blur) rounded once each, the ratio, the product, the L-term level sum
                    and the division by L: 5 + L roundings on |blur| * |ratio|."""
    L, G = len(parts), len(parts[0])
    scale = torch.zeros((G,) + tuple(parts[0][0][0].shape), dtype=torch.float64)
    depth = 0
    for l in range(L):
        for g in range(G):
            y, r, sb, K = parts[l][g]
            stat_err = sb.pow(2).mean().sqrt() if reduce == 'std' else sb.max()
            a = y.std(unbiased=False) if reduce == 'std' else y.max()
            rel = stat_err / a.abs() if float(a) != 0 else torch.zeros((), dtype=torch.float64)
            scale[g] += r.abs() * (sb + y.abs() * (rel + 1)) / L
            depth = max(depth, K + y.dim() - 2)
    return scale, depth + 5 + L
