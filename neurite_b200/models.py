"""
neurite_b200.models -- the SynthMorph / SynthSeg image generator of neurite
(adalca/neurite: neurite/tf/models.py:920-1301, labels_to_image_new) as a torch.nn.Module on CUDA tensors.

    gen = labels_to_image_new(labels_in=range(16), in_shape=(160, 192, 224))
    image, label_map = gen(labels)            # labels [B, *in_shape, 1], integer or float

Stages and where they run:
    velocity PerlinNoise -> VecInt(5) -> RescaleTransform(2) -> ComposeTransform -> nearest SpatialTransformer
                                              the existing layers
    crop, generation LUT, per-label means, exp(bias), max |image|     nrt_labels_to_image_f32 (one pass)
    GaussianNoise (+ background clearing)     nrt_philox_normal_f32 / nrt_philox_normal_background_f32
    random GaussianBlur, Subsample            utils.separable_conv, utils.gather_axis
    per-item min / max, normalisation, gamma  nrt_item_minmax_f32, nrt_norm_gamma_f32
    crop, output LUT, one-hot / int map       nrt_label_map_f32 / nrt_label_map_i32

Randomness.  Every component (warp, crop, mean, bias, noise, background, blur, slice, gamma) takes its seed from
`seeds` and draws with `seed + number of earlier calls`, like the layers; `seed=None` seeds from the operating
system.  An iterable of names seeds each with `hash(name)`, as the reference does; Python salts the hash of a
string per process (PYTHONHASHSEED), so such seeds repeat only within one process.  Small draws are made on the
host with numpy (crop, blur SDs, subsample); the tables (per-label mean U [B, C, N], background U [B], gamma
U [B, C]) are drawn on the device by the Philox stream of nrt_noise.cu, and TF's fp32 `u * (max - min) + min` is
applied in the kernel that reads them.  A call makes no device-to-host copy and leaves torch's RNG untouched.

A call is `_synthesize(labels, _draw(labels))`: `_draw` makes every random quantity (the plan), `_synthesize` is
deterministic given it.

Scope: the affine draw of the reference comes from voxelmorph (DrawAffineParams, draw_flip_matrix,
draw_swap_matrix) and is not built: non-zero aff_*, axes_flip, axes_swap and input_model raise
NotImplementedError.  The origin / center / scale matrices at identity affine are applied, so out_shape and
half_res work.
"""
import numpy as np
import torch

from . import augment, layers, utils
from ._lib import lib, check, ptr, stream_ptr, i32_array, require_cuda

_MAX_SEED = np.iinfo(int).max
_COMPONENTS = ('warp', 'crop', 'mean', 'bias', 'noise', 'background', 'blur', 'slice', 'gamma')


def _key(seed):
    return int(np.random.default_rng(seed).integers(_MAX_SEED))


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
        self._shift_cache = {}
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
        plan = {}
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
    def _affine_shift(self, device):
        """Dense shift of the identity affine with the origin / center / scale matrices, [1, *out_shape, N]."""
        key = (device.type, device.index)
        if key not in self._shift_cache:
            mat = torch.as_tensor(self.cfg['trans'][None, :self.cfg['num_dim'], :], dtype=torch.float32, device=device)
            st = layers.SpatialTransformer(shift_center=False)
            self._shift_cache[key] = st._affine_to_dense(mat, tuple(int(s) for s in self.cfg['out_shape']))
        return self._shift_cache[key]

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
        """labels [B, *in_shape, 1] -> the nearest-warped fp32 label map [B, *out_shape, 1] (and the shift)."""
        c = self.cfg
        x = labels if labels.dtype == torch.float32 else labels.to(torch.float32)
        B = x.shape[0]
        trans = self._affine_shift(x.device).expand(B, *self._affine_shift(x.device).shape[1:])
        def_field = None
        if plan['vel'] is not None:
            vel = plan['vel']
            if c['warp_zero_mean']:
                vel = vel - vel.mean(dim=tuple(range(1, c['num_dim'] + 1)), keepdim=True)
            def_field = layers.VecInt(int_steps=5)(vel)
            if not c['half_res']:
                def_field = layers.RescaleTransform(zoom_factor=2)(def_field)
            trans = layers.ComposeTransform()([trans, def_field])
        warped = layers.SpatialTransformer(interp_method='nearest', fill_value=0)([x, trans.contiguous()])
        return warped.contiguous(), def_field

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
            mnmx = utils._item_minmax(x2d) if c['normalize'] else None
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
            outputs.append(torch.eye(c['num_dim'] + 1, dtype=torch.float32, device=dev).expand(B, -1, -1).clone())
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
):
    """Build the module that augments label maps and synthesizes images from them (models.py:920-1301).  The
    arguments, defaults and outputs are the reference's; see the module docstring for the scope and the
    randomness.  Calling the module on a [B, *in_shape, 1] label map returns the outputs in the reference's
    order (the tensor itself when there is one)."""
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

    for name, v in (('aff_shift', aff_shift), ('aff_rotate', aff_rotate), ('aff_scale', aff_scale),
                    ('aff_shear', aff_shear)):
        if np.any(np.asarray(v) != 0):
            raise NotImplementedError(f'labels_to_image_new: {name} != 0 needs the voxelmorph affine draw, '
                                      f'which is not built')
    for t in ('shift', 'rot', 'scale', 'shear'):
        seeds.pop(t, None)
    origin = np.eye(num_dim + 1)
    origin[:num_dim, -1] = -0.5 * (in_shape - 1)
    center = np.eye(num_dim + 1)
    center[:num_dim, -1] = np.round(0.5 * (in_shape - (2 if half_res else 1) * out_shape))
    scale = np.diag((*[2 if half_res else 1] * num_dim, 1))
    trans = np.linalg.inv(origin) @ np.eye(num_dim + 1) @ origin @ center @ scale
    if axes_flip:
        raise NotImplementedError('labels_to_image_new: axes_flip needs voxelmorph.utils.draw_flip_matrix, '
                                  'which is not built')
    if axes_swap:
        assert all(x == out_shape[0] for x in out_shape), 'non-isotropic output shape'
        raise NotImplementedError('labels_to_image_new: axes_swap needs voxelmorph.utils.draw_swap_matrix, '
                                  'which is not built')

    used = {}
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

    cfg = dict(num_dim=num_dim, in_shape=in_shape, out_shape=out_shape, half_res=half_res, trans=trans,
               num_chan=int(num_chan), warp_min=warp_min, warp_max=warp_max, warp_blur_min=warp_blur_min,
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
