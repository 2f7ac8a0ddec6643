"""GPU tests of the generator's affine label warp: nrt_warp_labels_affine_f32 bit for bit against the oracle chain
and against the old three-stage chain built from the existing layers, the generator on the reference's affsynth_*
plans, determinism, the profiler's view, and full-size calls."""
import ast
import glob
import os
import zlib

import numpy as np
import pytest
import torch

import neurite_b200 as ne
from neurite_b200._lib import lib, check, ptr, stream_ptr, i32_array
from oracle import affine as oaff, noise as onoise, synth as osynth

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
F32 = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
AFFSYNTH = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLDEN, 'affsynth_*.npz')))


def _t(a):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV)


def _kernel(labels, mats, d, out_shape):
    """labels, mats, d device tensors -> nrt_warp_labels_affine_f32's output."""
    B, N = mats.shape[0], mats.shape[1]
    out = torch.empty(B, *out_shape, 1, device=DEV)
    check(lib.nrt_warp_labels_affine_f32(ptr(labels), ptr(mats), ptr(d), ptr(out), B, N,
                                         i32_array(labels.shape[1:-1]), i32_array(out_shape), stream_ptr(DEV)))
    return out


def _mats(kind, B, N, in_shape, out_shape, rng):
    """[B, N, N+1] fp32 warp matrices of one kind, each item its own."""
    half = kind == 'half_res'
    eye = np.eye(N + 1)
    aff = np.repeat(eye[None], B, 0)
    flip = swap = None
    if kind == 'int_shift':
        aff[:, :N, N] = rng.integers(-4, 5, (B, N))
    elif kind == 'half_shift':                                          # loc lands on .5: rint ties to even
        aff[:, :N, N] = rng.integers(-4, 5, (B, N)) + 0.5
    elif kind == 'rot90':
        r = 3 if N == 3 else 1
        p = np.zeros((B, 12 if N == 3 else 6), F32)
        p[:, N:N + r] = rng.choice([-180, -90, 90, 180], (B, r))
        aff = ne.models.affine_matrix(p, N).astype(np.float64)
    elif kind in ('random', 'half_res', 'flip', 'swap'):
        p = ne.models.affine_params(B, N, dict(shift=4, rot=180 if kind == 'random' else 30, scale=0.5, shear=0.3),
                                    dict(shift=False, rot=False, scale=False, shear=False),
                                    {k: int(rng.integers(1 << 30)) for k in ('shift', 'rot', 'scale', 'shear')})
        aff = ne.models.affine_matrix(p, N).astype(np.float64)
        if kind == 'flip':
            flip = ne.models.flip_matrix(np.arange(N) % 2 == 0, out_shape)
        if kind == 'swap':
            swap = ne.models.swap_matrix(np.roll(np.arange(N), 1))
    elif kind == 'far':                                                 # everything outside: fill
        aff[:, :N, N] = rng.choice([-1e5, 1e5], (B, N))
    m = oaff.compose(aff, in_shape, out_shape, half, flip, swap)[:, :N]
    return m.astype(F32)


CASES = [  # N, B, in_shape, out_shape, kind
    (3, 1, (9, 10, 13), (9, 10, 13), 'identity'),
    (3, 3, (9, 10, 13), (9, 10, 13), 'int_shift'),
    (3, 3, (8, 8, 8), (8, 8, 8), 'half_shift'),
    (3, 3, (12, 11, 10), (12, 11, 10), 'rot90'),
    (3, 3, (12, 11, 16), (7, 9, 6), 'random'),
    (3, 2, (12, 12, 16), (5, 5, 7), 'half_res'),
    (3, 2, (10, 12, 14), (10, 12, 14), 'flip'),
    (3, 3, (10, 10, 12), (10, 10, 10), 'swap'),
    (3, 2, (6, 7, 9), (6, 7, 9), 'far'),
    (2, 1, (17, 22), (17, 22), 'identity'),
    (2, 3, (17, 22), (17, 22), 'half_shift'),
    (2, 3, (16, 15), (16, 15), 'rot90'),
    (2, 3, (20, 23), (13, 16), 'random'),
    (2, 2, (20, 22), (9, 11), 'half_res'),
    (2, 2, (14, 14), (14, 14), 'swap'),
    (2, 2, (9, 12), (9, 12), 'far'),
]


@pytest.mark.parametrize('with_d', [False, True])
@pytest.mark.parametrize('N,B,in_shape,out_shape,kind', CASES)
def test_kernel_vs_oracle_chain(N, B, in_shape, out_shape, kind, with_d):
    rng = np.random.default_rng(zlib.crc32(repr((N, B, in_shape, kind, with_d)).encode()))
    labels = rng.integers(0, 16, (B, *in_shape, 1)).astype(F32)
    mats = _mats(kind, B, N, in_shape, out_shape, rng)
    d = None
    if with_d:
        d = rng.uniform(-3, 3, (B, *out_shape, N)).astype(F32)
        if kind == 'far':
            d[..., 0] = 1e6
        d[:, 0, 0] = np.round(d[:, 0, 0]) + 0.5                           # ties on the corner grid too
    dl, dm, dd = _t(labels), _t(mats), None if d is None else _t(d)
    got = _kernel(dl, dm, dd, out_shape).cpu().numpy()
    ref = oaff.warp_labels(labels, mats, d, out_shape)
    assert np.array_equal(got, ref) and not np.signbit(got).any()
    if kind == 'far':
        assert not got.any()


def test_kernel_unaligned_buffers_take_the_scalar_path():
    rng = np.random.default_rng(5)
    shape = (6, 7, 8)
    labels = rng.integers(0, 9, (2, *shape, 1)).astype(F32)
    mats = _mats('random', 2, 3, shape, shape, rng)
    d = rng.uniform(-2, 2, (2, *shape, 3)).astype(F32)
    buf = torch.zeros(d.size + 1, device=DEV)
    buf[1:] = _t(d).reshape(-1)
    dd = buf[1:].view(d.shape)                                           # 4 bytes past a 16-byte boundary
    out = torch.full((2 * int(np.prod(shape)) + 2,), -1.0, device=DEV)
    o = out[1:-1].view(2, *shape, 1)
    B, N = 2, 3
    dl, dm = _t(labels), _t(mats)
    check(lib.nrt_warp_labels_affine_f32(ptr(dl), ptr(dm), ptr(dd), ptr(o), B, N, i32_array(shape), i32_array(shape),
                                         stream_ptr(DEV)))
    assert np.array_equal(o.cpu().numpy(), oaff.warp_labels(labels, mats, d, shape))
    assert float(out[0]) == -1 and float(out[-1]) == -1


def test_kernel_rejects_bad_arguments():
    one = torch.zeros(4, device=DEV)
    s = i32_array([2, 2, 2])
    assert lib.nrt_warp_labels_affine_f32(ptr(one), ptr(one), None, ptr(one), 1, 4, s, s, stream_ptr(DEV)) != 0
    assert b'2 and 3' in lib.nrt_last_error_string()
    assert lib.nrt_warp_labels_affine_f32(None, ptr(one), None, ptr(one), 1, 3, s, s, stream_ptr(DEV)) != 0


# ---------------------------------------------------------------------------------------
# the old chain: dense shift (fixed order, eager torch ops) -> ComposeTransform -> nearest SpatialTransformer
# ---------------------------------------------------------------------------------------
def _dense_shift_torch(mats, out_shape):
    B, N = mats.shape[:2]
    grid = torch.meshgrid(*[torch.arange(s, dtype=torch.float32, device=DEV) for s in out_shape], indexing='ij')
    col = lambda i, k: mats[:, i, k].reshape(B, *[1] * N)                  # noqa: E731
    out = []
    for i in range(N):
        s = col(i, 0) * grid[0]
        for k in range(1, N):
            s = s + col(i, k) * grid[k]
        out.append((s + col(i, N)) - grid[i])
    return torch.stack(out, -1)


def _old_chain(labels, mats, d, out_shape):
    trans = _dense_shift_torch(mats, out_shape)
    if d is not None:
        trans = ne.layers.ComposeTransform()([trans, d])
    return ne.layers.SpatialTransformer(interp_method='nearest', fill_value=0)([labels, trans.contiguous()])


def _synthmorph_def(rng, shape):
    vel = torch.as_tensor(rng.uniform(-2, 2, (1, *[s // 2 for s in shape], 3)).astype(F32), device=DEV)
    return ne.layers.RescaleTransform(zoom_factor=2)(ne.layers.VecInt(int_steps=5)(vel)).contiguous()


@pytest.mark.parametrize('kind', ['identity', 'random'])
def test_full_size_kernel_vs_old_chain(kind):
    shape = (160, 192, 224)
    rng = np.random.default_rng(7)
    labels = torch.as_tensor(rng.integers(0, 16, (1, *shape, 1)).astype(F32), device=DEV)
    gen = ne.models.labels_to_image_new(range(16), in_shape=shape)
    aff = np.eye(4)[None]
    if kind == 'random':
        p = ne.models.affine_params(1, 3, dict(shift=30, rot=45, scale=0.1, shear=0.1),
                                    dict(shift=False, rot=False, scale=False, shear=False),
                                    dict(shift=1, rot=2, scale=3, shear=4))
        aff = ne.models.affine_matrix(p, 3)
    mats = _t(ne.models.compose_affine(aff, gen.cfg['aff_pre'], gen.cfg['aff_post']))
    d = _synthmorph_def(rng, shape)
    for dd in (None, d):
        got = _kernel(labels, mats, dd, shape)
        assert torch.equal(got, _old_chain(labels, mats, dd, shape))


# ---------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', AFFSYNTH)
def test_generator_on_affsynth_plan(name):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    kw = ast.literal_eval(str(fx['kwargs']))
    q = [fx['q%d' % i] for i in range(int(fx['nq']))]
    labels = fx['labels']
    c, p, aff = oaff.decode(kw, labels, q)
    gen = ne.models.labels_to_image_new(**dict(kw, vxm_affine=True, return_mean=True, return_vel=False,
                                                 return_def=False, return_bias=False))
    plan = {
        'aff': _t(aff['aff']),
        'trans': _t(fx['trans']),
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
    ref_outs = [fx['out%d' % i] for i in range(int(fx['nout']))]
    assert np.array_equal(outs[1].cpu().numpy(), ref_outs[1])                 # the reference's own label map
    if kw.get('return_aff'):
        i_aff = 2 + int(bool(kw.get('return_vel'))) + int(bool(kw.get('return_def')))
        assert np.array_equal(outs[2].cpu().numpy(), ref_outs[i_aff])         # return_aff: the drawn A
    if p['noise'] is not None:                  # the device draws Philox normals for keys (11, 12): the same z here
        u_sd = onoise.philox_uniform(11, p['mean_u'].shape[0] * c['num_chan'], 0, 1)
        p = dict(p, noise=(u_sd.reshape(-1, c['num_chan']), None))
    z = None
    if p['noise'] is not None:
        n = labels.shape[0] * int(np.prod(c['out_shape_eff'])) * c['num_chan']
        z = onoise.philox_normal64(12, n).reshape([labels.shape[0]] + c['out_shape_eff'] + [c['num_chan']])
    r = oaff.synth(labels, c, p, fx['trans'], z=z)
    assert np.array_equal(outs[-1].cpu().numpy(), r['mean'])                  # bit-exact uncorrupted mean
    lo, hi = osynth.image_interval(r, c, p, z)
    got = outs[0].cpu().numpy().astype(np.float64)
    assert np.all((got >= lo) & (got <= hi)), float(np.max(np.maximum(lo - got, got - hi)))


def _label_input(rng, B, shape, labels):
    return torch.as_tensor(rng.choice(np.asarray(labels), (B, *shape, 1)).astype(np.int32), device=DEV)


AFF_KW = dict(aff_shift=5, aff_rotate=30, aff_scale=0.1, aff_shear=0.1, axes_flip=True, axes_swap=True,
              vxm_affine=True)
AFF_SEEDS = {'shift': 11, 'rot': 12, 'scale': 13, 'shear': 14, 'flip': 15, 'swap': 16, 'warp': 1, 'mean': 3,
             'bias': 4, 'noise': 5, 'blur': 7, 'crop': 2, 'slice': 8, 'gamma': 9}


def test_generator_determinism_seed_calls_and_torch_rng_untouched():
    kw = dict(labels_in=range(4), in_shape=(12, 12, 12), return_aff=True, **AFF_KW)
    x = _label_input(np.random.default_rng(2), 2, (12, 12, 12), range(4))
    state, cstate = torch.get_rng_state(), torch.cuda.get_rng_state()
    a = ne.models.labels_to_image_new(seeds=AFF_SEEDS, **kw)(x)
    b = ne.models.labels_to_image_new(seeds=AFF_SEEDS, **kw)(x)
    assert torch.equal(torch.get_rng_state(), state) and torch.equal(torch.cuda.get_rng_state(), cstate)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    g = ne.models.labels_to_image_new(seeds=AFF_SEEDS, **kw)
    first, second = g(x), g(x)                                   # seed + calls: the second call draws afresh
    assert torch.equal(first[2], a[2]) and not torch.equal(second[2], first[2])
    # the drawn A is the host's draw from seed + calls
    for calls, out in ((0, first), (1, second)):
        p = ne.models.affine_params(2, 3, dict(shift=5, rot=30, scale=0.1, shear=0.1),
                                    dict(shift=False, rot=False, scale=False, shear=False),
                                    {k: AFF_SEEDS[k] + calls for k in ('shift', 'rot', 'scale', 'shear')})
        assert np.array_equal(out[2].cpu().numpy(), ne.models.affine_matrix(p, 3))
    # the label map is the oracle's warp of the plan's matrix
    plan = ne.models.labels_to_image_new(seeds=AFF_SEEDS, **kw)._draw(x)
    warped, d = g.warp_labels(x, plan)
    ref = oaff.warp_labels(x.cpu().numpy().astype(F32), plan['trans'].cpu().numpy(), d.cpu().numpy(), (12, 12, 12))
    assert np.array_equal(warped.cpu().numpy(), ref)


def _names(fn):
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    if not any(e.device_type == torch.autograd.DeviceType.CUDA for e in prof.events()):
        pytest.skip('torch.profiler recorded no CUDA events on this machine')
    return [e.name for e in prof.events()]


def test_profiler_kernel_and_no_device_to_host_copy():
    gen = ne.models.labels_to_image_new(range(8), in_shape=(16, 16, 16), seeds={'mean': 1}, **AFF_KW)
    x = _label_input(np.random.default_rng(4), 2, (16, 16, 16), range(8))
    gen(x)
    torch.cuda.synchronize()
    names = _names(lambda: gen(x))
    assert any('warp_labels_affine_kernel' in n for n in names)
    assert not any('DtoH' in n or 'Device -> Host' in n for n in names), [n for n in names if 'Memcpy' in n]
    plan = gen._draw(x)
    names = _names(lambda: gen.warp_labels(x, plan))
    assert any('warp_labels_affine_kernel' in n for n in names)
    assert not any('einsum' in n or 'bmm' in n or 'gemm' in n.lower() for n in names)


def test_full_size_synthmorph_bounds_vs_old_chain():
    shape = (160, 192, 224)
    gen = ne.models.labels_to_image_new(range(16), in_shape=shape, aff_shift=30, aff_rotate=45, aff_scale=0.1,
                                        aff_shear=0.1, axes_flip=True, vxm_affine=True,
                                        seeds={'mean': 1, 'warp': 2, 'shift': 3, 'rot': 4, 'scale': 5, 'shear': 6,
                                               'flip': 7})
    x = _label_input(np.random.default_rng(1), 1, shape, range(16))
    plan = gen._draw(x)
    image, onehot = gen._synthesize(x, plan)
    warped, d = gen.warp_labels(x, plan)
    assert torch.equal(warped, _old_chain(x.to(torch.float32), plan['trans'], d, shape))
    ref = torch.nn.functional.one_hot(warped[..., 0].to(torch.int64), 16).to(torch.float32)
    assert torch.equal(onehot, ref)
    assert float(image.min()) >= 0 and float(image.max()) <= 1


def test_swap_96_cubed_vs_oracle_chain():
    shape = (96, 96, 96)
    gen = ne.models.labels_to_image_new(range(8), in_shape=shape, aff_shift=10, aff_rotate=20, aff_scale=0.1,
                                        aff_shear=0.05, axes_swap=True, axes_flip=True, vxm_affine=True,
                                        seeds={'mean': 1, 'warp': 2, 'swap': 3, 'flip': 4})
    x = _label_input(np.random.default_rng(3), 1, shape, range(8))
    plan = gen._draw(x)
    warped, d = gen.warp_labels(x, plan)
    ref = oaff.warp_labels(x.cpu().numpy().astype(F32), plan['trans'].cpu().numpy(), d.cpu().numpy(), shape)
    assert np.array_equal(warped.cpu().numpy(), ref)
