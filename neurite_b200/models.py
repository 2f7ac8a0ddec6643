"""
neurite_b200.models -- the SynthMorph / SynthSeg image generator of neurite
(adalca/neurite: neurite/tf/models.py:920-1301, labels_to_image_new) as a torch.nn.Module on CUDA tensors.

    gen = labels_to_image_new(labels_in=range(16), in_shape=(160, 192, 224))
    image, label_map = gen(labels)            # labels [B, *in_shape, 1], integer or float

Stages and where they run:
    affine parameters, flip, swap, the composed [B, N, N+1] matrix     host (numpy), one copy to the device
    velocity PerlinNoise -> VecInt(5) -> RescaleTransform(2)          the existing layers
    dense affine shift, composition with the deformation, nearest label warp
                                              nrt_warp_labels_affine_f32 (one pass)
    crop, generation LUT, per-label means, exp(bias), max |image|     nrt_labels_to_image_f32 (one pass)
    GaussianNoise (+ background clearing)     nrt_philox_normal_f32 / nrt_philox_normal_background_f32
    random GaussianBlur, Subsample            utils.separable_conv, utils.gather_axis
    per-item min / max, normalisation, gamma  nrt_item_stats_f32, nrt_norm_gamma_f32
    crop, output LUT, one-hot / int map       nrt_label_map_f32 / nrt_label_map_i32

Randomness.  Every component (shift, rot, scale, shear, flip, swap, warp, crop, mean, bias, noise, background,
blur, slice, gamma) takes its seed from `seeds` and draws with `seed + number of earlier calls`, like the layers;
`seed=None` seeds from the operating system.  An iterable of names seeds each with `hash(name)`, as the reference
does; Python salts the hash of a string per process (PYTHONHASHSEED), so such seeds repeat only within one
process.  Small draws are made on the host with numpy (affine, flip, swap, crop, blur SDs, subsample); the tables
(per-label mean U [B, C, N], background U [B], gamma U [B, C]) are drawn on the device by the Philox stream of
nrt_noise.cu, and TF's fp32 `u * (max - min) + min` is applied in the kernel that reads them.  A call makes no
device-to-host copy and leaves torch's RNG untouched.

A call is `_synthesize(labels, _draw(labels))`: `_draw` makes every random quantity (the plan), `_synthesize` is
deterministic given it.

The affine.  The reference takes DrawAffineParams, ParamsToAffineMatrix, draw_flip_matrix and draw_swap_matrix
from voxelmorph; they are restated here as a contract (DESIGN.md §2): affine_params, affine_matrix, flip_matrix,
swap_matrix and compose_affine below, used when the builder is given vxm_affine=True.  Bounds must be scalars;
input_model raises NotImplementedError.
"""
import numpy as np
import torch

from . import _lib, augment, layers, utils
from ._lib import lib, check, ptr, stream_ptr, i32_array, require_cuda

_MAX_SEED = np.iinfo(int).max
_COMPONENTS = ('warp', 'crop', 'mean', 'bias', 'noise', 'background', 'blur', 'slice', 'gamma')
_AFFINE = ('shift', 'rot', 'scale', 'shear')
F32 = np.float32


def _key(seed):
    return int(np.random.default_rng(seed).integers(_MAX_SEED))


# ---- the affine draw (voxelmorph's DrawAffineParams, ParamsToAffineMatrix, draw_flip_matrix, draw_swap_matrix) ----
def affine_sizes(ndims):
    """Parameters per item and kind: shift N, rotation 3 (1 in 2-D), scale N, shear 3 (1 in 2-D)."""
    r = 3 if ndims == 3 else 1
    return {'shift': ndims, 'rot': r, 'scale': ndims, 'shear': r}


def affine_params(batch, ndims, bounds, normal, seeds):
    """[batch, 12] (3-D) or [batch, 6] (2-D) fp32 parameters, in the order shift, rotation (degrees), scale, shear.
    Each kind draws from numpy's generator seeded with seeds[kind]: uniform on [-bound, bound] as TF's fp32
    u * (2 bound) - bound, or with normal[kind] z * bound, the scale's z redrawn where |z| > 2 (truncated at 2 SD).
    A bound of 0 draws nothing and gives zeros."""
    out = []
    for kind, n in affine_sizes(ndims).items():
        b, shape = float(bounds[kind]), (batch, n)
        if b == 0:
            out.append(np.zeros(shape, F32))
            continue
        rng = np.random.default_rng(seeds.get(kind))
        if not normal[kind]:
            out.append((rng.random(shape, dtype=F32) * F32(2 * b) + F32(-b)).astype(F32))
            continue
        z = rng.standard_normal(shape, dtype=F32)
        while kind == 'scale' and np.any(np.abs(z) > 2):
            bad = np.abs(z) > 2
            z[bad] = rng.standard_normal(int(bad.sum()), dtype=F32)
        out.append((z * F32(b)).astype(F32))
    return np.concatenate(out, 1)


def affine_matrix(params, ndims):
    """ParamsToAffineMatrix(deg=True, shift_scale=True, last_row=True): [B, N+1, N+1] fp32 with A = R (Z S),
    Z = diag(1 + scale), S the upper unit-triangular shear, R = Rx (Ry Rz) in 3-D, and the shift as the last
    column; evaluated in fp64, rounded once."""
    p = np.asarray(params, np.float64)
    n = affine_sizes(ndims)
    shift, rot = p[:, :ndims], np.deg2rad(p[:, ndims:ndims + n['rot']])
    scale, shear = p[:, ndims + n['rot']:2 * ndims + n['rot']], p[:, 2 * ndims + n['rot']:]
    out = np.zeros((p.shape[0], ndims + 1, ndims + 1))
    for b in range(p.shape[0]):
        c, s = np.cos(rot[b]), np.sin(rot[b])
        if ndims == 3:
            rx = np.array([[1, 0, 0], [0, c[0], -s[0]], [0, s[0], c[0]]])
            ry = np.array([[c[1], 0, s[1]], [0, 1, 0], [-s[1], 0, c[1]]])
            rz = np.array([[c[2], -s[2], 0], [s[2], c[2], 0], [0, 0, 1]])
            r = rx @ (ry @ rz)
            sh = np.array([[1, shear[b, 0], shear[b, 1]], [0, 1, shear[b, 2]], [0, 0, 1]])
        else:
            r = np.array([[c[0], -s[0]], [s[0], c[0]]])
            sh = np.array([[1, shear[b, 0]], [0, 1]])
        out[b, :ndims, :ndims] = r @ (np.diag(1 + scale[b]) @ sh)
        out[b, :ndims, ndims] = shift[b]
        out[b, ndims, ndims] = 1
    return out.astype(F32)


def draw_flip(seed, ndims):
    """The flipped axes [ndims] bool: each with probability 1/2 (U[0, 1) > 0.5)."""
    return np.random.default_rng(seed).random(ndims, dtype=F32) > 0.5


def draw_swap(seed, ndims):
    """A uniformly random permutation of the axes."""
    return np.random.default_rng(seed).permutation(ndims)


def flip_matrix(flip, out_shape):
    """draw_flip_matrix(out_shape, shift_center=False) given the flipped axes: x -> (out_shape - 1) - x there."""
    n = len(out_shape)
    m = np.eye(n + 1)
    for a in np.flatnonzero(flip):
        m[a, a], m[a, n] = -1, out_shape[a] - 1
    return m


def swap_matrix(perm):
    """draw_swap_matrix given the permutation: P[i, perm[i]] = 1."""
    n = len(perm)
    m = np.eye(n + 1)
    m[:n, :n] = np.eye(n)[list(perm)]
    return m


def compose_affine(aff, pre, post, flip=None, swap=None):
    """The matrix the warp applies (models.py:1117-1131): (((pre @ aff) @ post) @ flip) @ swap in fp64, top N rows
    as fp32 [B, N, N+1].  pre = inv(origin), post = origin @ center @ scale."""
    m = pre @ np.asarray(aff, np.float64) @ post
    for f in (flip, swap):
        if f is not None:
            m = m @ f
    n = m.shape[-1] - 1
    return np.ascontiguousarray(m[:, :n, :]).astype(F32)


def _uniform01(key, shape, device):
    """Philox U(0, 1] table of `shape` on the device (nrt_philox_uniform_f32 with lo = 0, hi = 1: exact u)."""
    out = torch.empty(shape, dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        check(lib.nrt_philox_uniform_f32(key, out.numel(), 0.0, 1.0, ptr(out), stream_ptr(device)))
    return out


def generation_lut(labels_in):
    """(labels_in as a dict, generation labels, LUT input label -> generation index), models.py:1172-1178."""
    if not isinstance(labels_in, dict):
        labels_in = {i: i for i in labels_in}
    labels_gen = set(labels_in.values())
    ind = {gen: i for i, gen in enumerate(labels_gen)}
    lut = [ind.get(labels_in.get(i), 0) for i in range(max(labels_in) + 1)]
    return labels_in, labels_gen, lut


def output_lut(labels_in, labels_out, one_hot):
    """(LUT or None when the reference skips the gather, number of output labels), models.py:1265-1279."""
    lut = list(labels_in) if labels_out is None else labels_out
    if not isinstance(lut, dict):
        lut = {i: i for i in lut}
    labels_out = set(lut.values())
    if one_hot:
        ind = {out: i for i, out in enumerate(labels_out)}
        lut = {inp: ind[out] for inp, out in lut.items()}
    if any(k != lut[k] for k in lut) or set(labels_in) - set(lut):
        return [lut.get(i, -1 if one_hot else 0) for i in range(max(labels_in) + 1)], len(labels_out)
    return None, len(labels_out)


class LabelsToImage(torch.nn.Module):
    """The generator labels_to_image_new returns; see the module docstring."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self._calls = 0
        self._ident_dev = {}
        c = cfg
        N = c['num_dim']
        self.vel_layer = None
        if c['warp_max'] > 0:
            self.vel_layer = layers.PerlinNoise(
                shape=(*(c['out_shape'] // (1 if c['half_res'] else 2)), N), noise_min=c['warp_min'],
                noise_max=c['warp_max'], isotropic=False, fwhm_min=np.asarray(c['warp_blur_min']) / 2,
                fwhm_max=np.asarray(c['warp_blur_max']) / 2, reduce='max', axes=-1, seed=c['seeds'].get('warp'))
        self.bias_layer = None
        if c['bias_max'] > 0:
            div = 2 if c['half_res'] else 1
            self.bias_layer = layers.PerlinNoise(
                noise_min=c['bias_min'], noise_max=c['bias_max'], isotropic=False,
                fwhm_min=c['bias_blur_min'] / div, fwhm_max=c['bias_blur_max'] / div, reduce='max',
                seed=c['seeds'].get('bias'))
        self.crop_layer = layers.RandomCrop(crop_min=c['crop_min'], crop_max=c['crop_max'], prob=c['crop_prob'],
                                            axis=c['crop_axes'], seed=c['seeds'].get('crop'))
        self.crop_layer.build((None, *c['out_shape'], 1))
        blur = layers.GaussianBlur(sigma=c['blur_max'], min_sigma=c['blur_min'], random=True)
        blur.build((None, *c['out_shape'], c['num_chan']))
        self._blur_sigma, self._blur_min = blur.sigma, blur.min_sigma
        div = 2 if c['half_res'] else 1
        self.slice_layer = layers.Subsample(prob=c['slice_prob'], stride_min=max(1, c['slice_stride_min'] / div),
                                            stride_max=max(1, c['slice_stride_max'] / div), axes=c['slice_axes'])
        self.slice_layer.build((None, *c['out_shape'], c['num_chan']))
        self._lut_dev = {}

    # ---- the draws ----
    def _seed(self, name):
        s = self.cfg['seeds'].get(name)
        return None if s is None else s + self._calls

    def _draw(self, labels):
        """Every random quantity of one call -> plan (dict)."""
        c = self.cfg
        require_cuda(labels)
        dev = labels.device
        B, C, Nl = labels.shape[0], c['num_chan'], len(c['labels_gen'])
        out_shape = [int(s) for s in c['out_shape']]
        N = c['num_dim']
        plan = {}
        if any(v != 0 for v in c['aff_bounds'].values()) or c['axes_flip'] or c['axes_swap']:
            params = affine_params(B, N, c['aff_bounds'], c['aff_normal'], {t: self._seed(t) for t in _AFFINE})
            aff = affine_matrix(params, N)
            flip = swap = None
            if c['axes_flip']:       # one matrix per call, shared by the batch
                flip = flip_matrix(draw_flip(self._seed('flip'), N), out_shape)
            if c['axes_swap']:
                swap = swap_matrix(draw_swap(self._seed('swap'), N))
            trans = compose_affine(aff, c['aff_pre'], c['aff_post'], flip, swap)
            # both matrices in one pinned buffer and one asynchronous copy: the host does not wait for the stream
            host = torch.from_numpy(np.concatenate([aff.ravel(), trans.ravel()])).pin_memory()
            mats = host.to(dev, non_blocking=True)
            plan['aff'] = mats[:aff.size].view(B, N + 1, N + 1)
            plan['trans'] = mats[aff.size:].view(B, N, N + 1)
        else:                        # nothing random: the identity's matrices, cached on the device
            plan['aff'], plan['trans'] = self._identity(dev, B)
        plan['vel'] = self.vel_layer(labels) if self.vel_layer is not None else None
        plan['crop'] = None
        if c['crop_prob'] != 0:
            plan['crop'] = self.crop_layer._draw([B, *out_shape, 1])
        plan['mean_u'] = _uniform01(_key(self._seed('mean')), (B, C, Nl), dev)
        plan['bias'] = None
        if self.bias_layer is not None:
            plan['bias'] = self.bias_layer(torch.zeros((), device=dev).expand(B, *out_shape, C))
        plan['noise'] = None
        if c['noise_max'] != 0:
            rand = np.random.default_rng(self._seed('noise'))
            plan['noise'] = (int(rand.integers(_MAX_SEED)), int(rand.integers(_MAX_SEED)))
        plan['bg_u'] = _uniform01(_key(self._seed('background')), (B,), dev) if c['zero_background'] > 0 else None
        plan['blur'] = None
        if any(s > 0 for s in self._blur_sigma):
            # GaussianBlur(random=True) -> utils.gaussian_kernel(random=True): the SDs and the window
            eps = np.finfo(np.float32).eps
            sig = [max(f, eps) for f in self._blur_sigma]
            mins = [max(f, eps) for f in self._blur_min]
            gen = torch.Generator().manual_seed(int(np.random.default_rng(self._seed('blur')).integers(2 ** 31)))
            drawn = [float(a + (b - a) * torch.rand(1, generator=gen).item()) for a, b in zip(mins, sig)]
            plan['blur'] = (drawn, [float(np.round(f * 3) * 2 + 1) for f in sig])
        plan['slice'] = None
        sl = self.slice_layer
        if not (sl.prob == 0 or sl.stride_max == 1):
            # Subsample -> utils.subsample_axis: the axis, the thickness and the Bernoulli draw
            rand = np.random.default_rng(self._seed('slice'))
            ax = list(sl.axes)[int(rand.integers(0, len(sl.axes)))]
            thick = np.float32(rand.uniform(sl.stride_min, sl.stride_max))
            if sl.prob < 1 and not (rand.uniform() < sl.prob):
                thick = np.float32(1)
            plan['slice'] = (ax, utils.subsample_indices(out_shape[ax - 1], thick, sl.upsample))
        plan['gamma_u'] = _uniform01(_key(self._seed('gamma')), (B, C), dev) if c['gamma'] > 0 else None
        self._calls += 1
        return plan

    # ---- the deterministic rest ----
    def _identity(self, device, batch):
        """The identity affine [B, N+1, N+1] and its warp matrix (origin, center and scale only) [B, N, N+1], on
        the device."""
        key = (device.type, device.index, batch)
        if key not in self._ident_dev:
            c = self.cfg
            eye = np.repeat(np.eye(c['num_dim'] + 1, dtype=F32)[None], batch, 0)
            self._ident_dev[key] = (torch.as_tensor(eye, device=device),
                                    torch.as_tensor(compose_affine(eye, c['aff_pre'], c['aff_post']), device=device))
        return self._ident_dev[key]

    def _luts(self, device):
        key = (device.type, device.index)
        if key not in self._lut_dev:
            c = self.cfg
            t = lambda v: torch.as_tensor(np.asarray(v, np.float32), device=device)   # noqa: E731
            gen = torch.as_tensor(np.asarray(c['gen_lut'], np.int32), device=device)
            out = None if c['out_lut'] is None else torch.as_tensor(np.asarray(c['out_lut'], np.int32), device=device)
            self._lut_dev[key] = (gen, out, t(c['mean_min']), t(c['mean_max']))
        return self._lut_dev[key]

    def warp_labels(self, labels, plan):
        """labels [B, *in_shape, 1] -> (the nearest-warped fp32 label map [B, *out_shape, 1], the deformation or
        None).  The affine is plan['trans'] [B, N, N+1]; a plan without it warps with the identity affine."""
        c = self.cfg
        x = (labels if labels.dtype == torch.float32 else labels.to(torch.float32)).contiguous()
        B, N = x.shape[0], c['num_dim']
        mats = plan.get('trans')
        mats = self._identity(x.device, B)[1] if mats is None else mats.contiguous()
        def_field = d = None
        if plan['vel'] is not None:
            vel = plan['vel']
            if c['warp_zero_mean']:
                vel = vel - vel.mean(dim=tuple(range(1, N + 1)), keepdim=True)
            def_field = layers.VecInt(int_steps=5)(vel)
            if not c['half_res']:
                def_field = layers.RescaleTransform(zoom_factor=2)(def_field)
            d = def_field.contiguous()
        out_shape = [int(s) for s in c['out_shape']]
        warped = torch.empty(B, *out_shape, 1, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            check(lib.nrt_warp_labels_affine_f32(ptr(x), ptr(mats), ptr(d), ptr(warped), B, N,
                                                 i32_array(x.shape[1:-1]), i32_array(out_shape),
                                                 stream_ptr(x.device)))
        return warped, def_field

    def _crop_args(self, plan):
        out_shape = [int(s) for s in self.cfg['out_shape']]
        if plan['crop'] is None:
            return 1, 1, 0, 1
        ax, lo, hi = plan['crop']
        return out_shape[ax - 1], int(np.prod(out_shape[ax:], dtype=np.int64)), lo, hi

    def _synthesize(self, labels, plan):
        c = self.cfg
        require_cuda(labels)
        dev = labels.device
        warped, def_field = self.warp_labels(labels, plan)
        B, C = warped.shape[0], c['num_chan']
        out_shape = [int(s) for s in c['out_shape']]
        V = int(np.prod(out_shape, dtype=np.int64))
        crop = self._crop_args(plan)
        gen_lut, out_lut, mmin, mmax = self._luts(dev)
        st = stream_ptr(dev)

        # labels -> intensities (* bias), max |image|
        bias, apply_exp = plan['bias'], 1
        if bias is not None:
            if c['bias_func'] is not torch.exp:
                bias, apply_exp = c['bias_func'](bias).to(torch.float32), 0
            bias = bias.contiguous()
        image = torch.empty(B, *out_shape, C, dtype=torch.float32, device=dev)
        want_mean, want_bias = c['return_mean'] and bias is not None, c['return_bias'] and bias is not None
        mean = torch.empty_like(image) if want_mean else None
        bias_out = torch.empty_like(image) if want_bias else None
        absmax = torch.empty(1, dtype=torch.float32, device=dev)
        nb = lib.nrt_labels_to_image_workspace_bytes()
        ws = utils._scratch(dev, nb)
        with torch.cuda.device(dev):
            check(lib.nrt_labels_to_image_f32(ptr(warped), B, V, C, *crop, ptr(gen_lut), gen_lut.numel(),
                                              len(c['labels_gen']), ptr(plan['mean_u']), ptr(mmin), ptr(mmax),
                                              ptr(bias), apply_exp, ptr(image), ptr(mean), ptr(bias_out),
                                              ptr(absmax), ptr(ws), nb, st))
        if mean is None:
            mean = image

        # GaussianNoise(noise_min, noise_max): SD U[min, max] per (item, channel), relative to max |image|;
        # with zero_background, fused with the background clearing
        if plan['noise'] is not None or plan['bg_u'] is not None:
            table = torch.zeros(B * C, dtype=torch.float32, device=dev)
            k_sd, k_noise = plan['noise'] if plan['noise'] is not None else (0, 0)
            noisy = torch.empty_like(image)
            with torch.cuda.device(dev):
                if plan['noise'] is not None:
                    check(lib.nrt_philox_uniform_f32(k_sd, B * C, float(c['noise_min']), float(c['noise_max']),
                                                     ptr(table), st))
                if plan['bg_u'] is None:
                    shape = [B, *out_shape, C]
                    sd_shape = [B] + [1] * len(out_shape) + [C]
                    check(lib.nrt_philox_normal_f32(k_noise, i32_array(shape), i32_array(sd_shape), len(shape),
                                                    ptr(table), ptr(absmax), ptr(image), ptr(noisy), st))
                else:
                    check(lib.nrt_philox_normal_background_f32(k_noise, B, V, C, ptr(table), ptr(absmax), ptr(image),
                                                               ptr(warped), *crop, ptr(plan['bg_u']),
                                                               float(c['zero_background']), ptr(noisy), st))
            image = noisy

        if plan['blur'] is not None:
            sig, win = plan['blur']
            k = utils.gaussian_kernel(sigma=sig, windowsize=win, separate=True)
            k = k if isinstance(k, list) else [k]
            # every tap in one pinned buffer and one asynchronous copy: the host does not wait for the stream
            taps = torch.cat(k).pin_memory().to(dev, non_blocking=True)
            offs = np.cumsum([0] + [t.numel() for t in k])
            image = utils.separable_conv(image, [taps[a:b] for a, b in zip(offs[:-1], offs[1:])], batched=True)
        if plan['slice'] is not None:
            ax, index = plan['slice']
            image = utils.gather_axis(image, index, ax)

        if c['normalize'] or plan['gamma_u'] is not None:
            x2d = image.contiguous().reshape(B, -1)
            mnmx = utils._item_stats(x2d, _lib.NRT_STAT_MINMAX) if c['normalize'] else None
            image = utils._norm_gamma(x2d, C, mnmx, plan['gamma_u'], c['gamma']).reshape(image.shape)

        # output label map
        if c['one_hot']:
            label_map = torch.empty(B, *out_shape, c['num_out'], dtype=torch.float32, device=dev)
            fn, extra = lib.nrt_label_map_f32, (c['num_out'],)
        else:
            label_map = torch.empty(B, *out_shape, 1, dtype=torch.int32, device=dev)
            fn, extra = lib.nrt_label_map_i32, ()
        with torch.cuda.device(dev):
            check(fn(ptr(warped), B, V, *crop, ptr(out_lut), 0 if out_lut is None else out_lut.numel(), *extra,
                     ptr(label_map), st))

        outputs = []
        if c['return_im']:
            outputs.append(image)
        if c['return_map']:
            outputs.append(label_map)
        if c['return_vel']:
            outputs.append(plan['vel'])
        if c['return_def']:
            outputs.append(def_field)
        if c['return_aff']:
            aff = plan.get('aff')
            if aff is None:
                aff = torch.eye(c['num_dim'] + 1, dtype=torch.float32, device=dev).expand(B, -1, -1)
            outputs.append(aff.clone())
        if c['return_mean']:
            outputs.append(mean)
        if c['return_bias']:
            outputs.append(bias_out if bias_out is not None else torch.exp(plan['bias']))
        return outputs[0] if len(outputs) == 1 else outputs

    def forward(self, labels):
        return self._synthesize(labels, self._draw(labels))


def labels_to_image_new(
    labels_in,
    labels_out=None,
    in_shape=None,
    out_shape=None,
    input_model=None,
    num_chan=1,
    aff_shift=0,
    aff_rotate=0,
    aff_scale=0,
    aff_shear=0,
    aff_normal_shift=False,
    aff_normal_rotate=False,
    aff_normal_scale=False,
    aff_normal_shear=False,
    axes_flip=False,
    axes_swap=False,
    warp_min=0.01,
    warp_max=2,
    warp_blur_min=(8, 8),
    warp_blur_max=(32, 32),
    warp_zero_mean=False,
    crop_min=0,
    crop_max=0.2,
    crop_prob=0,
    crop_axes=None,
    mean_min=None,
    mean_max=None,
    noise_min=0.1,
    noise_max=0.2,
    zero_background=0,
    blur_min=0,
    blur_max=1,
    bias_min=0.01,
    bias_max=0.1,
    bias_blur_min=32,
    bias_blur_max=64,
    bias_func=torch.exp,
    slice_stride_min=1,
    slice_stride_max=8,
    slice_prob=0,
    slice_axes=None,
    normalize=True,
    gamma=0.5,
    one_hot=True,
    half_res=False,
    seeds={},
    return_im=True,
    return_map=True,
    return_vel=False,
    return_def=False,
    return_aff=False,
    return_mean=False,
    return_bias=False,
    id=0,
    vxm_affine=False,
):
    """Build the module that augments label maps and synthesizes images from them (models.py:920-1301).  The
    arguments, defaults and outputs are the reference's; see the module docstring for the randomness.  Calling
    the module on a [B, *in_shape, 1] label map returns the outputs in the reference's order (the tensor itself
    when there is one).

    Affine augmentation (vxm_affine=True).  The reference draws the affine with voxelmorph, which is not part of
    it; this package restates those pieces (DrawAffineParams, ParamsToAffineMatrix, draw_flip_matrix,
    draw_swap_matrix) as a contract, and vxm_affine=True says the caller wants that restatement.  Without it,
    non-zero aff_*, axes_flip and axes_swap raise NotImplementedError naming the argument, as before.  With it,
    each item draws its own shift (voxels), rotation (degrees), scale (added to 1) and shear, uniform on
    [-aff_*, aff_*], or normal with aff_* as the SD when aff_normal_* is set (the scale truncated at 2 SD).
    axes_flip flips each axis with probability 1/2 and axes_swap permutes the axes (isotropic out_shape only);
    both draw one matrix per call for the whole batch.  return_aff returns the drawn [B, N+1, N+1] matrix.
    The bounds must be scalars; input_model raises NotImplementedError."""
    if isinstance(seeds, str):
        seeds = [seeds]
    if isinstance(seeds, dict):
        seeds = seeds.copy()
    if not isinstance(seeds, dict):
        seeds = {f: hash(f) for f in seeds}

    if input_model is not None:
        raise NotImplementedError('labels_to_image_new: input_model is not built')
    in_shape = np.asarray(in_shape)
    if out_shape is None:
        out_shape = in_shape
    out_shape = np.array(out_shape) // (2 if half_res else 1)
    num_dim = len(in_shape)

    aff_bounds = {'shift': aff_shift, 'rot': aff_rotate, 'scale': aff_scale, 'shear': aff_shear}
    aff_normal = {'shift': aff_normal_shift, 'rot': aff_normal_rotate, 'scale': aff_normal_scale,
                  'shear': aff_normal_shear}
    for name, v in zip(('aff_shift', 'aff_rotate', 'aff_scale', 'aff_shear'), aff_bounds.values()):
        if np.ndim(v) != 0:
            raise NotImplementedError(f'labels_to_image_new: {name} must be a scalar bound')
        if v != 0 and not vxm_affine:
            raise NotImplementedError(f'labels_to_image_new: {name} != 0 needs the restated voxelmorph affine '
                                      f'draw; pass vxm_affine=True')
    used = {t: seeds.pop(t, None) for t in _AFFINE}
    origin = np.eye(num_dim + 1)
    origin[:num_dim, -1] = -0.5 * (in_shape - 1)
    center = np.eye(num_dim + 1)
    center[:num_dim, -1] = np.round(0.5 * (in_shape - (2 if half_res else 1) * out_shape))
    scale = np.diag((*[2 if half_res else 1] * num_dim, 1))
    if axes_flip:
        if not vxm_affine:
            raise NotImplementedError('labels_to_image_new: axes_flip needs the restated voxelmorph '
                                      'draw_flip_matrix; pass vxm_affine=True')
        used['flip'] = seeds.pop('flip', None)
    if axes_swap:
        assert all(x == out_shape[0] for x in out_shape), 'non-isotropic output shape'
        if not vxm_affine:
            raise NotImplementedError('labels_to_image_new: axes_swap needs the restated voxelmorph '
                                      'draw_swap_matrix; pass vxm_affine=True')
        used['swap'] = seeds.pop('swap', None)

    for name in _COMPONENTS:
        active = {'warp': warp_max > 0, 'bias': bias_max > 0, 'background': zero_background > 0,
                  'gamma': gamma > 0}.get(name, True)
        if active:
            used[name] = seeds.pop(name, None)

    labels_in, labels_gen, gen_lut = generation_lut(labels_in)
    num_label = len(labels_gen)
    if mean_min is None:
        mean_min = [0] * num_label
    if mean_max is None:
        mean_max = [1] * num_label
    # bounds broadcast against the [B, C, N] draw like tf.random.uniform's minval / maxval: [N] or [C, N]
    mean_min = np.broadcast_to(np.asarray(mean_min, np.float32), (int(num_chan), num_label)).copy()
    mean_max = np.broadcast_to(np.asarray(mean_max, np.float32), (int(num_chan), num_label)).copy()

    if gamma > 0:
        assert 0 < gamma < 1, f'gamma value {gamma} outside interval [0, 1)'
    out_lut, num_out = output_lut(labels_in, labels_out, one_hot)

    if return_vel and not warp_max > 0:
        raise NameError("labels_to_image_new: return_vel needs warp_max > 0 (no 'vel_field')")
    if return_def and not warp_max > 0:
        raise NameError("labels_to_image_new: return_def needs warp_max > 0 (no 'def_field')")
    if return_bias and not bias_max > 0:
        raise NameError("labels_to_image_new: return_bias needs bias_max > 0 (no 'bias_field')")
    assert not seeds, f'unknown seeds {seeds}'

    cfg = dict(num_dim=num_dim, in_shape=in_shape, out_shape=out_shape, half_res=half_res,
               aff_bounds=aff_bounds, aff_normal=aff_normal, axes_flip=bool(axes_flip), axes_swap=bool(axes_swap),
               aff_pre=np.linalg.inv(origin), aff_post=origin @ center @ scale, num_chan=int(num_chan),
               warp_min=warp_min, warp_max=warp_max, warp_blur_min=warp_blur_min,
               warp_blur_max=warp_blur_max, warp_zero_mean=warp_zero_mean, crop_min=crop_min, crop_max=crop_max,
               crop_prob=crop_prob, crop_axes=crop_axes, mean_min=mean_min, mean_max=mean_max, noise_min=noise_min,
               noise_max=noise_max, zero_background=zero_background, blur_min=blur_min, blur_max=blur_max,
               bias_min=bias_min, bias_max=bias_max, bias_blur_min=bias_blur_min, bias_blur_max=bias_blur_max,
               bias_func=bias_func, slice_stride_min=slice_stride_min, slice_stride_max=slice_stride_max,
               slice_prob=slice_prob, slice_axes=slice_axes, normalize=normalize, gamma=gamma, one_hot=one_hot,
               seeds=used, labels_gen=labels_gen, gen_lut=gen_lut, out_lut=out_lut, num_out=num_out,
               return_im=return_im, return_map=return_map, return_vel=return_vel, return_def=return_def,
               return_aff=return_aff, return_mean=return_mean, return_bias=return_bias, id=id)
    return LabelsToImage(cfg)
