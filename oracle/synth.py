"""
The label-to-image stages of labels_to_image_new.  TEST INFRASTRUCTURE (see oracle/__init__.py).

    crop_mask_bruteforce              draw_crop_mask's mask (augment.py:280-284) element by element in fp32
    labels_to_image                   models.py:1163-1216 on a warped fp32 label map: crop, generation LUT, per-label
                                      means u * (max - min) + min, image = mean * exp(bias); fp32, one rounding per op
    noise_background                  models.py:1219-1231: x + z * (sd * scale), then * keep
    norm_gamma                        minmax_norm per item (utils.py:953-968), then pow(x, u * (hi - lo) + lo)
    label_map                         models.py:1276-1282: crop, output LUT, one-hot or int map
    crop_window                       RandomCrop: x * mask on one axis

Provenance: contract for tf.range's fp32 length and element formula (neurite_b200.augment.tf_range_f32) and for
TF's GPU gather giving 0 at an out-of-range index.  exp and pow are evaluated by numpy in fp32 here; the device's
expf / powf differ from them by a few ulp, so those stages are compared within a bound, every other stage bit
for bit.
"""
import numpy as np

F32 = np.float32


def crop_mask_bruteforce(width, prop_low, prop_cen):
    delta = F32(F32(1) / F32(width))
    n = int(np.ceil(F32(F32(1) / delta)))
    prop = np.array([F32(F32(i) * delta) for i in range(n)], F32)
    return (prop >= F32(prop_low)) & (prop < F32(F32(prop_low) + F32(prop_cen)))


def crop_labels(warped, crop, out_shape):
    """warped [B, *out_shape, 1] fp32 -> int32 labels with the crop (axis, lo, hi) applied (0 outside)."""
    lab = np.trunc(np.asarray(warped, F32)).astype(np.int32)
    if crop is not None:
        ax, lo, hi = crop
        idx = np.arange(lab.shape[ax])
        keep = (idx >= lo) & (idx < hi)
        shp = [1] * lab.ndim
        shp[ax] = lab.shape[ax]
        lab = lab * keep.reshape(shp).astype(np.int32)
    return lab


def gather0(lut, idx):
    """tf.gather on the GPU: 0 for an index outside [0, len(lut))."""
    lut = np.asarray(lut, np.int32)
    ok = (idx >= 0) & (idx < lut.size)
    return np.where(ok, lut[np.clip(idx, 0, lut.size - 1)], 0).astype(np.int32)


def labels_to_image(lab, gen_lut, u, mean_min, mean_max, bias=None, bias_fn=np.exp):
    """lab [B, *S, 1] int32 (cropped), u [B, C, N], bounds [N] or [C, N] -> (image, mean) [B, *S, C] fp32."""
    idx = gather0(gen_lut, lab[..., 0])                                   # [B, *S]
    mn, mx = np.asarray(mean_min, F32), np.asarray(mean_max, F32)
    d = (mx - mn).astype(F32)
    B, C = u.shape[:2]
    mean = np.empty(idx.shape + (C,), F32)
    for b in range(B):
        for c in range(C):
            i = idx[b]
            dc, mc = np.broadcast_to(d, (C,) + d.shape[-1:])[c], np.broadcast_to(mn, (C,) + mn.shape[-1:])[c]
            mean[b, ..., c] = (u[b, c][i] * dc[i]).astype(F32) + mc[i]
    mean = mean.astype(F32)
    if bias is None:
        return mean, mean
    f = bias_fn(np.asarray(bias, F32)).astype(F32) if bias_fn is not None else np.asarray(bias, F32)
    return (mean * f).astype(F32), mean


def noise_background(x, z, sd, scale, lab, bg_u, zero_background):
    """x [B, *S, C], z the normals [B, *S, C], sd [B, C] -> (x + z * (sd * scale)) * keep."""
    B, C = sd.shape
    s = (np.asarray(sd, F32) * F32(scale)).astype(F32).reshape((B,) + (1,) * (x.ndim - 2) + (C,))
    y = (x + (np.asarray(z, F32) * s).astype(F32)).astype(F32)
    if bg_u is None:
        return y
    clear = (lab[..., 0] == 0) & (np.asarray(bg_u, F32).reshape((B,) + (1,) * (x.ndim - 2)) < F32(zero_background))
    return (y * (~clear).astype(F32)[..., None]).astype(F32)


def norm_gamma(x, normalize=True, gamma_u=None, gamma=0.0):
    """Per item b: div_no_nan(x - min, max - min), then pow(., u[b, c] * (hi - lo) + lo) with lo, hi = 1 -+ gamma."""
    x = np.asarray(x, F32)
    out = np.empty_like(x)
    for b in range(x.shape[0]):
        y = x[b]
        if normalize:
            mn, mx = F32(y.min()), F32(y.max())
            d = F32(mx - mn)
            y = np.zeros_like(y) if d == 0 else ((y - mn).astype(F32) / d).astype(F32)
        if gamma_u is not None:
            lo, hi = F32(1 - gamma), F32(1 + gamma)
            g = (np.asarray(gamma_u[b], F32) * F32(hi - lo)).astype(F32) + lo
            y = np.power(y, g.astype(F32)).astype(F32)
        out[b] = y
    return out


def label_map(lab, out_lut, one_hot, num_out):
    """lab [B, *S, 1] int32 (cropped) -> one-hot [B, *S, M] fp32 or int32 [B, *S, 1]."""
    l = lab[..., 0] if out_lut is None else gather0(out_lut, lab[..., 0])
    if not one_hot:
        return l[..., None].astype(np.int32)
    return (l[..., None] == np.arange(num_out)).astype(F32)


def crop_window(x, axis, lo, hi):
    x = np.asarray(x)
    idx = np.arange(x.shape[axis])
    shp = [1] * x.ndim
    shp[axis] = x.shape[axis]
    m = ((idx >= lo) & (idx < hi)).reshape(shp)
    if x.dtype == np.float32:
        return (x * m.astype(F32)).astype(F32)
    return np.where(m, x, 0).astype(x.dtype)


# ---------------------------------------------------------------------------------------
# the whole generator given its draws (tests/golden/synth_*, crop_*, minmax_*)
# ---------------------------------------------------------------------------------------
def _uni(u, lo, hi):
    """TF's fp32 u * (hi - lo) + lo on a raw U[0, 1) draw."""
    lo, hi = np.asarray(lo, F32), np.asarray(hi, F32)
    return (np.asarray(u, F32) * (hi - lo).astype(F32) + lo).astype(F32)


def crop_from_draws(q, k, shape, crop_min, crop_max, axis, prob, bilateral):
    """draw_crop_mask (augment.py:246-287) on the replayed draws q[k:] -> ((axis, lo, hi), k)."""
    ndim = len(shape)
    axis = [axis] if np.isscalar(axis) else (list(range(ndim)) if axis is None else list(axis))
    axis = sorted({a + ndim if a < 0 else a for a in axis})
    prop_cut = F32(crop_max)
    if crop_min < crop_max:
        prop_cut = _uni(q[k], crop_min, crop_max).reshape(())
        k += 1
    if prob < 1:
        prop_cut = F32(prop_cut * F32(np.asarray(q[k], F32).reshape(()) < F32(prob)))
        k += 1
    rp = np.asarray(q[k], F32).reshape(())
    k += 1
    if not bilateral:
        rp = F32(rp < F32(0.5))
    pl, pc = F32(prop_cut * rp), F32(F32(1) - prop_cut)
    ax = axis[int(np.asarray(q[k]).reshape(()))]
    k += 1
    mask = crop_mask_bruteforce(shape[ax], pl, pc)
    assert mask.size == shape[ax], 'tf.range length != width: the reference reshape fails'
    idx = np.flatnonzero(mask)
    lo, hi = (int(idx[0]), int(idx[-1]) + 1) if idx.size else (0, 0)
    return (ax, lo, hi), k


def _perlin(q, k, G, gshape, nmin, nmax, fmin, fmax, reduce):
    """PerlinNoise draws of G items (per item, per level: SD table, noise, one SD per spatial axis) -> fields."""
    from . import noise as onoise
    fmin, fmax = list(np.ravel(fmin)), list(np.ravel(fmax))
    L, D = len(fmin), len(gshape) - 2
    noise = np.zeros([L, G] + list(gshape), F32)
    sig = [[None] * G for _ in range(L)]
    for g in range(G):
        for l in range(L):
            noise[l, g] = (np.asarray(q[k + 1], F32) * _uni(q[k], nmin, nmax)).astype(F32)
            sig[l][g] = [onoise.sigma_from_draw(u, fmin[l] / 2.355, fmax[l] / 2.355) for u in q[k + 2:k + 2 + D]]
            k += 2 + D
    out = onoise.perlin_from_draws(noise, sig, [f / 2.355 for f in fmax], reduce)
    return out.reshape([G] + list(gshape[1:])), k


def generation_lut(labels_in):
    if not isinstance(labels_in, dict):
        labels_in = {i: i for i in labels_in}
    labels_gen = set(labels_in.values())
    ind = {gen: i for i, gen in enumerate(labels_gen)}
    return labels_in, labels_gen, [ind.get(labels_in.get(i), 0) for i in range(max(labels_in) + 1)]


def output_lut(labels_in, labels_out, one_hot):
    lut = list(labels_in) if labels_out is None else labels_out
    if not isinstance(lut, dict):
        lut = {i: i for i in lut}
    out = set(lut.values())
    if one_hot:
        ind = {o: i for i, o in enumerate(out)}
        lut = {i: ind[o] for i, o in lut.items()}
    if any(k != lut[k] for k in lut) or set(labels_in) - set(lut):
        return [lut.get(i, -1 if one_hot else 0) for i in range(max(labels_in) + 1)], len(out)
    return None, len(out)


SYNTH_DEFAULTS = dict(labels_out=None, out_shape=None, num_chan=1, warp_min=0.01, warp_max=2, warp_blur_min=(8, 8),
                      warp_blur_max=(32, 32), crop_min=0, crop_max=0.2, crop_prob=0, crop_axes=None, mean_min=None,
                      mean_max=None, noise_min=0.1, noise_max=0.2, zero_background=0, blur_min=0, blur_max=1,
                      bias_min=0.01, bias_max=0.1, bias_blur_min=32, bias_blur_max=64, slice_stride_min=1,
                      slice_stride_max=8, slice_prob=0, slice_axes=None, normalize=True, gamma=0.5, one_hot=True,
                      half_res=False)


def decode_synth(kwargs, labels, q):
    """A synth_* fixture's arguments, label map and draw queue -> (cfg, plan): every random quantity in numpy.
    plan: vel [B, *vs, N] | None, crop (axis, lo, hi) | None, mean_u [B, C, N], bias [B, *S, C] | None,
    noise (u_sd [B, C], z [B, *S, C]) | None, bg_u [B] | None, blur [N] fp32 SDs | None, slice (axis, thick) |
    None, gamma_u [B, C] | None."""
    c = dict(SYNTH_DEFAULTS, **kwargs)
    B = labels.shape[0]
    in_shape = np.asarray(c['in_shape'])
    out_shape = np.array(in_shape if c['out_shape'] is None else c['out_shape']) // (2 if c['half_res'] else 1)
    N, C = len(in_shape), c['num_chan']
    c['out_shape_eff'] = [int(s) for s in out_shape]
    labels_in, gen, c['gen_lut'] = generation_lut(c['labels_in'])
    c['num_label'] = len(gen)
    c['out_lut'], c['num_out'] = output_lut(labels_in, c['labels_out'], c['one_hot'])
    S = c['out_shape_eff']
    p, k = {}, 0
    p['vel'] = None
    if c['warp_max'] > 0:
        vs = [int(s) for s in out_shape // (1 if c['half_res'] else 2)]
        p['vel'], k = _perlin(q, k, B, [1] + vs + [N], c['warp_min'], c['warp_max'],
                              np.asarray(c['warp_blur_min']) / 2, np.asarray(c['warp_blur_max']) / 2, 'max')
    p['crop'] = None
    if c['crop_prob'] != 0:
        axes = list(range(1, N + 1)) if c['crop_axes'] is None else c['crop_axes']
        p['crop'], k = crop_from_draws(q, k, [B] + S + [1], c['crop_min'], c['crop_max'], axes, c['crop_prob'], False)
    p['mean_u'] = np.asarray(q[k], F32).reshape(B, C, c['num_label'])
    k += 1
    p['bias'] = None
    if c['bias_max'] > 0:
        div = 2 if c['half_res'] else 1
        p['bias'], k = _perlin(q, k, B, [1] + S + [C], c['bias_min'], c['bias_max'], c['bias_blur_min'] / div,
                               c['bias_blur_max'] / div, 'max')
    p['noise'] = None
    if c['noise_max'] != 0:
        p['noise'] = (np.asarray(q[k], F32).reshape(B, C), np.asarray(q[k + 1], F32).reshape([B] + S + [C]))
        k += 2
    p['bg_u'] = None
    if c['zero_background'] > 0:
        p['bg_u'] = np.asarray(q[k], F32).reshape(B)
        k += 1
    sig = np.ravel(c['blur_max']).tolist()
    sig = sig * N if len(sig) == 1 else sig
    mins = np.ravel(c['blur_min']).tolist()
    mins = mins * N if len(mins) == 1 else mins
    p['blur'] = None
    if any(s > 0 for s in sig):
        eps = np.finfo(F32).eps
        p['blur'] = ([_uni(q[k + i], max(a, eps), max(b, eps)).reshape(()) for i, (a, b) in enumerate(zip(mins, sig))],
                     [float(np.round(max(b, eps) * 3) * 2 + 1) for b in sig])
        k += N
    p['slice'] = None
    div = 2 if c['half_res'] else 1
    smin, smax = max(1, c['slice_stride_min'] / div), max(1, c['slice_stride_max'] / div)
    if not (c['slice_prob'] == 0 or smax == 1):
        axes = list(range(1, N + 1)) if c['slice_axes'] is None else [int(a) % (N + 2) for a in np.ravel(c['slice_axes'])]
        ax = axes[int(np.asarray(q[k]).reshape(()))]
        thick = _uni(q[k + 1], smin, smax).reshape(())
        k += 2
        if c['slice_prob'] < 1:
            bit = np.asarray(q[k], F32).reshape(()) < F32(c['slice_prob'])
            thick = F32(F32(thick * F32(bit)) + F32(not bit))
            k += 1
        p['slice'] = (ax, thick)
    p['gamma_u'] = None
    if c['gamma'] > 0:
        p['gamma_u'] = np.asarray(q[k], F32).reshape(B, C)
        k += 1
    assert k == len(q), 'draw queue not consumed: %d of %d' % (k, len(q))
    return c, p


def affine_shift(c):
    """The dense shift of the identity affine with the origin / center / scale matrices, [*S, N] fp32."""
    in_shape = np.asarray(c['in_shape'])
    S = c['out_shape_eff']
    n = len(S)
    center = np.round(0.5 * (in_shape - (2 if c['half_res'] else 1) * np.asarray(S)))
    s = 2 if c['half_res'] else 1
    grid = np.stack(np.meshgrid(*[np.arange(v, dtype=F32) for v in S], indexing='ij'), -1)
    return ((grid * F32(s) + center.astype(F32)).astype(F32) - grid).astype(F32)


def synth_from_plan(labels, c, p, z=None):
    """labels_to_image_new on the plan, numpy fp32, one rounding per TF op -> dict of the stages and outputs.
    z: the normals of the noise stage (plan['noise'][1] by default)."""
    from . import interp as ointerp, conv as oconv
    B, N, C = labels.shape[0], len(c['in_shape']), c['num_chan']
    S = c['out_shape_eff']
    trans = np.broadcast_to(affine_shift(c), [B] + S + [N]).astype(F32)
    r = {}
    if p['vel'] is not None:
        d = ointerp.vec_int(p['vel'], int_steps=5)
        if not c['half_res']:
            d = ointerp.rescale_transform(d, 2)
        r['def'] = d
        trans = np.stack([ointerp.compose([trans[b], d[b]]) for b in range(B)], 0)
    warped = ointerp.spatial_transformer(labels.astype(F32), trans, 'nearest', fill_value=0).astype(F32)
    lab = crop_labels(warped, p['crop'], S)
    r['warped'], r['lab'] = warped, lab
    mmin = [0] * c['num_label'] if c['mean_min'] is None else c['mean_min']
    mmax = [1] * c['num_label'] if c['mean_max'] is None else c['mean_max']
    image, mean = labels_to_image(lab, c['gen_lut'], p['mean_u'], mmin, mmax, p['bias'])
    r['mean'] = mean
    if p['bias'] is not None:
        r['bias'] = np.exp(p['bias']).astype(F32)
    r['pre_noise'] = image
    if p['noise'] is not None:
        u_sd, zz = p['noise']
        sd = _uni(u_sd, c['noise_min'], c['noise_max'])
        scale = F32(np.max(np.abs(image)))
        zz = zz if z is None else z
        s = (sd * scale).astype(F32).reshape((B,) + (1,) * N + (C,))
        image = (image + ((np.asarray(zz, F32) * s).astype(F32) + F32(0)).astype(F32)).astype(F32)
    if p['bg_u'] is not None:
        clear = (lab[..., 0] == 0) & (p['bg_u'].reshape((B,) + (1,) * N) < F32(c['zero_background']))
        image = (image * (~clear).astype(F32)[..., None]).astype(F32)
    r['pre_blur'] = image
    if p['blur'] is not None:
        sig, win = p['blur']
        ks = [oconv.gaussian_kernel([float(s)], windowsize=[w], separate=True) for s, w in zip(sig, win)]
        image = oconv.separable_conv(image, ks, batched=True)
    if p['slice'] is not None:
        image = oconv.subsample_axis(image, p['slice'][0], p['slice'][1])
    r['pre_norm'] = image
    image = norm_gamma(image, c['normalize'], p['gamma_u'], c['gamma'] if p['gamma_u'] is not None else 0.0)
    r['image'] = image
    r['map'] = label_map(lab, c['out_lut'], c['one_hot'], c['num_out'])
    return r


def synth_outputs(kwargs, r, p):
    """The reference's outputs in its order from synth_from_plan's stages."""
    c = dict(SYNTH_DEFAULTS, return_im=True, return_map=True, return_vel=False, return_def=False, return_aff=False,
             return_mean=False, return_bias=False)
    c.update(kwargs)
    out = []
    for key, v in (('return_im', r['image']), ('return_map', r['map']), ('return_vel', p['vel']),
                   ('return_def', r.get('def')), ('return_mean', r['mean']), ('return_bias', r.get('bias'))):
        if c[key]:
            out.append(v)
    return out


def minmax_norm(x, axis=None):
    """utils.py:953-968 in fp32: div_no_nan(x - min, max - min) over `axis`."""
    x = np.asarray(x, F32)
    mn = np.min(x, axis=axis, keepdims=True)
    mx = np.max(x, axis=axis, keepdims=True)
    d = (mx - mn).astype(F32)
    out = np.zeros(np.broadcast(x, d).shape, F32)
    np.divide((x - mn).astype(F32), d, out=out, where=(d != 0))
    return out


def image_interval(r, c, p, z=None):
    """An interval [lo, hi] (float64) that holds every fp32 evaluation of the image for the plan, by a device or by
    synth_from_plan, given the stages `r` of synth_from_plan:
      intensities   expf (2 ulp on the device, numpy's within 1) and the product: 5 * 2^-23 |image| (0 without bias)
      noise         Box-Muller within NORMAL_REL |z| (oracle/noise.py), z rounded to fp32, the SD * scale product and
                    the scale's own error (the intensity bound at the maximum), then the sum's rounding
      blur          per pass: the incoming error blurred with |k| plus 4 K 2^-24 (|k| * |x|) (oracle/noise.py's bound)
      normalise     an interval, not a linearisation: the item's min and max move by at most the largest error E,
                    so (x - mn) / (mx - mn) lies in [(x - e - mn - E)+ / (mx - mn + 2E), (x + e - mn + E) /
                    (mx - mn - 2E)], clipped to [0, 1], widened by the subtraction and division roundings
      gamma         pow is increasing on [0, inf) for gamma > 0: the interval's ends to the power gamma (the same fp32
                    gamma on both sides), widened by 8 * 2^-23 for powf
    """
    from . import conv as oconv, noise as onoise
    u = 2.0 ** -24
    B, N, C = r['lab'].shape[0], len(c['in_shape']), c['num_chan']
    x = r['pre_noise'].astype(np.float64)
    e = 10 * u * np.abs(x) if p['bias'] is not None else np.zeros_like(x)
    if p['noise'] is not None:
        u_sd, zz = p['noise']
        zz = zz if z is None else z
        sd = _uni(u_sd, c['noise_min'], c['noise_max']).astype(np.float64).reshape((B,) + (1,) * N + (C,))
        scale = float(np.max(np.abs(x)))
        az = np.abs(np.asarray(zz, np.float64))
        x = x + az * 0                         # shape only
        n_abs = az * sd * scale
        e = e + n_abs * (onoise.NORMAL_REL + 6 * u) + az * sd * float(np.max(e)) + 2 * u * (np.abs(x) + n_abs)
    if p['bg_u'] is not None:
        clear = (r['lab'][..., 0] == 0) & (p['bg_u'].reshape((B,) + (1,) * N) < F32(c['zero_background']))
        e = e * (~clear)[..., None]
    xv = r['pre_blur'].astype(np.float64)
    if p['blur'] is not None:
        sig, win = p['blur']
        ks = [oconv.gaussian_kernel([float(s)], windowsize=[w], separate=True) for s, w in zip(sig, win)]
        for a, k in enumerate(ks):
            ak = np.abs(np.asarray(k, np.float64))
            e = oconv.conv1d_axis(e, ak, a + 1).astype(np.float64) * 1.001 + \
                4 * (k.size + 1) * u * oconv.conv1d_axis(np.abs(xv), ak, a + 1).astype(np.float64) * 1.001
            xv = oconv.conv1d_axis(xv, k, a + 1).astype(np.float64)
    if p['slice'] is not None:
        e = oconv.subsample_axis(e, p['slice'][0], p['slice'][1])
    x0 = r['pre_norm'].astype(np.float64)
    lo, hi = x0 - e, x0 + e
    if c['normalize']:
        for b in range(B):
            E = float(np.max(e[b]))
            mn, mx = float(x0[b].min()), float(x0[b].max())
            if mx == mn and E == 0:
                lo[b], hi[b] = 0, 0
                continue
            num_lo = np.maximum(x0[b] - e[b] - mn - E, 0)
            num_hi = x0[b] + e[b] - mn + E
            lo[b] = np.clip(num_lo / (mx - mn + 2 * E) * (1 - 4 * u) - u, 0, 1)
            hi[b] = np.clip(num_hi / max(mx - mn - 2 * E, 1e-30) * (1 + 4 * u) + u, 0, 1)
    if p['gamma_u'] is not None:
        g = _uni(p['gamma_u'], F32(1 - c['gamma']), F32(1 + c['gamma'])).astype(np.float64).reshape(
            (B,) + (1,) * N + (C,))
        lo = np.power(np.maximum(lo, 0), g) * (1 - 16 * u)
        hi = np.power(np.maximum(hi, 0), g) * (1 + 16 * u) + u
    return lo - u, hi + u
