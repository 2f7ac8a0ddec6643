"""
GPU parity tests for the SURVEY.md 8f-3 / 8f-4 rows: MutualInformation (fused soft
quantisation + tensor-core joint histogram), soft_quantize, GaussianBlur / separable_conv,
Subsample.  Through the public python API -> ctypes -> the C ABI, against tests/golden (the
reference's own source on tools/tfshim.py) and the numpy oracle.

Tolerances: MI 1e-5 relative (+2e-6 absolute: the metric is a difference of logs) -- TF's
matmul / reduction order is unspecified; convolutions 1e-5 (tap order unspecified in TF);
gaussian_kernel, subsample gathers and soft_quantize(return_log=True) are bit-exact.
"""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from oracle import conv as oconv, mi as omi
from test_oracle_mi_conv import SEPCONV_KW

pytestmark = pytest.mark.gpu
F32 = np.float32
MI_TOL = dict(rtol=1e-5, atol=2e-6)


def dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.fixture(scope='module')
def ne(cuda):
    import neurite_b200
    return neurite_b200


# ------------------------------------------------------------------ soft_quantize
@pytest.mark.parametrize('name', golden_names('softq_'))
def test_soft_quantize_golden(ne, name):
    g = load_golden(name)
    kw = eval(str(g['kw']), {'array': np.array, 'float32': np.float32, 'dtype': np.dtype})
    out = ne.utils.soft_quantize(dev(g['x']), **kw).cpu().numpy()
    assert out.shape == g['out'].shape
    if kw.get('return_log'):
        np.testing.assert_array_equal(out, g['out'])
    else:
        np.testing.assert_allclose(out, g['out'], rtol=3e-6, atol=1e-30)


# ------------------------------------------------------------------ MutualInformation
@pytest.mark.parametrize('generic', [False, True])
@pytest.mark.parametrize('name', golden_names('mi_volumes_'))
def test_mi_volumes_golden(ne, monkeypatch, name, generic):
    if generic:
        monkeypatch.setenv('NRT_MI_GENERIC', '1')
    g = load_golden(name)
    kw = dict(nb_bins=int(g['nb_bins']))
    if 'min_clip' in g.files:
        kw.update(soft_bin_alpha=float(g['alpha']), min_clip=float(g['min_clip']), max_clip=float(g['max_clip']))
    m = ne.metrics.MutualInformation(**kw)
    assert np.float32(m.soft_bin_alpha) == np.float32(g['alpha'])
    x, y = dev(g['x']), dev(g['y'])
    np.testing.assert_allclose(m.volumes(x, y).cpu().numpy(), g['mi'], **MI_TOL)
    if 'mi_self' in g.files:
        np.testing.assert_allclose(m.volumes(x, x).cpu().numpy(), g['mi_self'], **MI_TOL)


@pytest.mark.parametrize('generic', [False, True])
def test_mi_channelwise_segs_volume_seg_golden(ne, monkeypatch, generic):
    if generic:
        monkeypatch.setenv('NRT_MI_GENERIC', '1')
    g = load_golden('mi_channelwise_c3')
    out = ne.metrics.MutualInformation().channelwise(dev(g['x']), dev(g['y'])).cpu().numpy()
    assert out.shape == g['mi'].shape
    np.testing.assert_allclose(out, g['mi'], **MI_TOL)
    for L in (16, 5):
        g = load_golden('mi_segs_L%d' % L)
        np.testing.assert_allclose(ne.metrics.MutualInformation().segs(dev(g['x']), dev(g['y'])).cpu().numpy(),
                                   g['mi'], **MI_TOL)
    g = load_golden('mi_volume_seg')
    m = ne.losses.MutualInformation(nb_bins=16)
    np.testing.assert_allclose(m.volume_seg(dev(g['vol']), dev(g['seg'])).cpu().numpy(), g['mi_vs'], **MI_TOL)
    np.testing.assert_allclose(m.volume_seg(dev(g['seg']), dev(g['vol'])).cpu().numpy(), g['mi_sv'], **MI_TOL)


def test_mi_errors(ne):
    Err = ne.metrics.InvalidArgumentError
    rng = np.random.default_rng(0)
    v = dev(rng.uniform(0, 1, (2, 4, 5, 1)).astype(F32))
    p = dev(rng.uniform(0, 1, (2, 4, 5, 16)).astype(F32))
    with pytest.raises(Err, match='two single-channel'):
        ne.metrics.MutualInformation().volumes(p, p)
    with pytest.raises(Err):
        ne.metrics.MutualInformation().maps(p, p[..., :3])
    with pytest.raises(Err):
        ne.metrics.MutualInformation().maps(p, -p)
    with pytest.raises(Err, match='multi-channel'):
        ne.metrics.MutualInformation().volume_seg(v, v)
    with pytest.raises(Err):
        ne.metrics.MutualInformation(nb_bins=16).volume_seg(v, p[..., :5])
    with pytest.raises(Err, match='do not match'):
        ne.metrics.MutualInformation().channelwise(p, p[:, :3])
    with pytest.raises(AssertionError):
        ne.metrics.MutualInformation(bin_centers=np.linspace(0, 1, 4), nb_bins=4)


@pytest.mark.parametrize('nb', [16, 24, 32, 48])
def test_mi_vs_oracle_ragged_sizes_and_explicit_centers(ne, nb):
    """voxel counts that are not multiples of the 8/16/32-voxel MMA chunks, bins that are not
    multiples of 8, explicit bin centres (the reference cannot run those; the oracle can)."""
    rng = np.random.default_rng(nb)
    for V in (1, 7, 33, 1000, 4099):
        x = rng.uniform(0, 1, (2, V, 1)).astype(F32)
        y = np.clip(x * 0.5 + 0.3 * rng.uniform(0, 1, x.shape), 0, 1).astype(F32)
        out = ne.metrics.MutualInformation(nb_bins=nb).volumes(dev(x), dev(y)).cpu().numpy()
        np.testing.assert_allclose(out, omi.MutualInformation(nb_bins=nb).volumes(x, y), **MI_TOL)
    centers = np.sort(rng.uniform(0, 1, nb - 3)).astype(F32)
    kw = dict(bin_centers=centers, soft_bin_alpha=80.0)
    out = ne.metrics.MutualInformation(**kw).volumes(dev(x), dev(y)).cpu().numpy()
    np.testing.assert_allclose(out, omi.MutualInformation(**kw).volumes(x, y), **MI_TOL)
    # maps with nb labels
    lx = rng.standard_normal((2, 777, nb)).astype(F32)
    px = np.exp(lx) / np.exp(lx).sum(-1, keepdims=True)
    py = np.roll(px, 1, axis=-1) * 0.5 + 0.5 * px
    out = ne.metrics.MutualInformation().maps(dev(px.astype(F32)), dev(py.astype(F32))).cpu().numpy()
    np.testing.assert_allclose(out, omi.MutualInformation().maps(px.astype(F32), py.astype(F32)), **MI_TOL)


def test_mi_full_size_volume_pair_properties_and_mid_size_oracle(ne, monkeypatch):
    """BASELINE.json's 160x192x224 volume: tensor-core path == CUDA-core path, symmetry,
    MI(x,x) > MI(x,y) > 0; and a 64x96x112 pair against the oracle."""
    gen = torch.Generator('cuda').manual_seed(1)
    for S, with_oracle in (((160, 192, 224), False), ((64, 96, 112), True)):
        x = torch.rand((2,) + S + (1,), device='cuda', generator=gen)
        y = (0.7 * x ** 2 + 0.1 + 0.1 * torch.rand(x.shape, device='cuda', generator=gen)).clamp_(0, 1)
        m = ne.metrics.MutualInformation(nb_bins=16)
        a, b, s = m.volumes(x, y).cpu().numpy(), m.volumes(y, x).cpu().numpy(), m.volumes(x, x).cpu().numpy()
        np.testing.assert_allclose(a, b, rtol=1e-5)
        assert np.all(s > a) and np.all(a > 0.3)
        monkeypatch.setenv('NRT_MI_GENERIC', '1')
        c = m.volumes(x, y).cpu().numpy()
        monkeypatch.delenv('NRT_MI_GENERIC')
        np.testing.assert_allclose(a, c, rtol=1e-5)
        if with_oracle:
            ref = omi.MutualInformation(nb_bins=16).volumes(x.cpu().numpy(), y.cpu().numpy())
            np.testing.assert_allclose(a, ref, **MI_TOL)


# ------------------------------------------------------------------ gaussian kernel / blur / separable conv
@pytest.mark.parametrize('name', golden_names('gausskernel_'))
def test_gaussian_kernel_golden_bit_exact(ne, name):
    g = load_golden(name)
    sigma = g['sigma'].tolist()
    if name.endswith('2d_full'):
        np.testing.assert_array_equal(ne.utils.gaussian_kernel(sigma).numpy(), g['k'])
        return
    ks = ne.utils.gaussian_kernel(sigma, separate=True)
    ks = ks if isinstance(ks, list) else [ks]
    for i, k in enumerate(ks):
        np.testing.assert_array_equal(k.numpy(), g['k%d' % i])


@pytest.mark.parametrize('generic', [False, True])
@pytest.mark.parametrize('name', golden_names('blur'))
def test_gaussian_blur_golden(ne, monkeypatch, name, generic):
    if generic is True:
        monkeypatch.setenv('NRT_CONV_GENERIC', '1')
    g = load_golden(name)
    sigma = g['sigma'].tolist()
    lay = ne.layers.GaussianBlur(sigma=sigma)
    out = lay(dev(g['x'])).cpu().numpy()
    assert out.shape == g['out'].shape
    np.testing.assert_allclose(out, g['out'], rtol=1e-5, atol=1e-6)
    assert lay.get_config()['sigma'] == lay.sigma


@pytest.mark.parametrize('name', golden_names('sepconv_'))
def test_separable_conv_golden(ne, name):
    g = load_golden(name)
    kw = SEPCONV_KW[str(g['kw'])](g)
    kw['kernels'] = [torch.from_numpy(k) for k in kw['kernels']] if isinstance(kw['kernels'], list) \
        else torch.from_numpy(kw['kernels'])
    out = ne.utils.separable_conv(dev(g['x']), **kw).cpu().numpy()
    assert out.shape == g['out'].shape
    # random (not normalised) kernels, outputs up to ~20 in magnitude with cancellation: absolute floor 1e-5
    np.testing.assert_allclose(out, g['out'], rtol=1e-5, atol=1e-5)


def test_blur_shapes_kernels_and_paths_vs_oracle(ne):
    """column pass (inner >= 32) / row pass (inner < 32, C = 1 and 3), wide kernels, ragged sizes, anisotropic and
    zero sigmas."""
    rng = np.random.default_rng(21)
    for shape, sigma in (((1, 70, 33, 45, 1), 1.0), ((2, 13, 20, 37, 3), [2.0, 0.6, 1.4]), ((1, 5, 130, 1), 4.0),
                         ((1, 40, 41, 2), [0.0, 5.0]), ((3, 300, 1), 9.0), ((1, 20, 20, 20, 1), 6.5),
                         ((2, 9, 17, 70, 1), [0.5, 2.3, 1.0]), ((1, 64, 30, 129, 1), [1.5, 0.0, 0.7]),
                         ((3, 5, 4, 3, 1), 2.0), ((1, 100, 16, 64, 1), 0.7)):
        x = rng.standard_normal(shape).astype(F32)
        ref = oconv.gaussian_blur(x, sigma)
        out = ne.layers.GaussianBlur(sigma=sigma)(dev(x)).cpu().numpy()
        np.testing.assert_allclose(out, ref, rtol=1e-5, atol=2e-6)
    # identity: all sigmas zero returns the input object
    t = dev(x)
    assert ne.layers.GaussianBlur(sigma=0)(t) is t


def test_blur_full_size_properties(ne):
    """160x192x224: constant stays constant away from the border (kernel sums to 1), the blur
    is linear, an impulse reproduces the outer product of the 1-D kernels."""
    S = (160, 192, 224)
    lay = ne.layers.GaussianBlur(sigma=[1.0, 2.0, 1.5])
    ks = [k.numpy() for k in ne.utils.gaussian_kernel([1.0, 2.0, 1.5], separate=True)]
    one = torch.ones((1,) + S + (1,), device='cuda')
    out = lay(one)[0, 8:-8, 8:-8, 8:-8, 0]
    assert float((out - 1).abs().max()) < 2e-6
    imp = torch.zeros((1,) + S + (1,), device='cuda')
    imp[0, 80, 96, 112, 0] = 1
    o = lay(imp)[0, ..., 0]
    r = [len(k) // 2 for k in ks]
    box = o[80 - r[0]:81 + r[0], 96 - r[1]:97 + r[1], 112 - r[2]:113 + r[2]].cpu().numpy()
    np.testing.assert_allclose(box, np.einsum('i,j,k->ijk', *ks), rtol=1e-5, atol=1e-9)
    assert abs(float(o.sum()) - 1) < 1e-5
    a = torch.randn((1,) + S + (1,), device='cuda')
    b = torch.randn_like(a)
    np.testing.assert_allclose(lay(a + 2 * b).cpu().numpy(), (lay(a) + 2 * lay(b)).cpu().numpy(), rtol=0, atol=2e-5)


def test_separable_conv_gradient(ne):
    rng = np.random.default_rng(31)
    x = torch.from_numpy(rng.standard_normal((2, 6, 40, 7, 2)).astype(F32)).cuda().requires_grad_(True)
    ks = [torch.from_numpy(rng.standard_normal(n).astype(F32)) for n in (3, 4, 5)]
    for padding in ('SAME', 'VALID'):
        y = ne.utils.separable_conv(x, ks, batched=True, padding=padding)
        w = torch.randn_like(y)
        (g,) = torch.autograd.grad((y * w).sum(), x)
        xd = x.detach().double().cpu().requires_grad_(True)
        t = xd.permute(0, 4, 1, 2, 3).reshape(-1, 1, 6, 40, 7)
        for ax, k in enumerate(ks):
            shape = [1, 1, 1, 1, 1]
            shape[2 + ax] = k.numel()
            if padding == 'SAME':
                tot = k.numel() - 1
                pads = [0, 0] * (2 - ax) + [tot // 2, tot - tot // 2] + [0, 0] * ax
                t = torch.nn.functional.pad(t, pads)
            t = torch.nn.functional.conv3d(t, k.double().reshape(shape))
        yr = t.reshape(2, 2, *t.shape[2:]).permute(0, 2, 3, 4, 1)
        np.testing.assert_allclose(y.detach().cpu().numpy(), yr.detach().numpy(), rtol=1e-5, atol=1e-5)
        (gr,) = torch.autograd.grad((yr * w.double().cpu()).sum(), xd)
        np.testing.assert_allclose(g.cpu().numpy(), gr.numpy(), rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------ Subsample
def test_subsample_vs_oracle(ne):
    rng = np.random.default_rng(41)
    x = rng.standard_normal((2, 12, 15, 18, 2)).astype(F32)
    for ax in (1, 2, 3):
        for thick in (1.0, 2.4, 5.0):
            for up in (True, False):
                idx = ne.utils.subsample_indices(x.shape[ax], thick, up)
                np.testing.assert_array_equal(idx, oconv.subsample_indices(x.shape[ax], thick, up))
                out = ne.utils.gather_axis(dev(x), idx, ax).cpu().numpy()
                np.testing.assert_array_equal(out, oconv.subsample_axis(x, ax, thick, up))
    lay = ne.layers.Subsample(stride_min=2, stride_max=4, seed=3)
    out = lay(dev(x))
    assert out.shape == x.shape and lay.axes == [1, 2, 3]
    # every output slice along the drawn axis is a copy of an input slice
    outn = out.cpu().numpy()
    hit = [all(any(np.array_equal(np.take(outn, i, ax), np.take(x, j, ax)) for j in range(x.shape[ax]))
               for i in range(x.shape[ax])) for ax in (1, 2, 3)]
    assert any(hit)
    assert ne.layers.Subsample(stride_max=1)(dev(x)).shape == x.shape


# ------------------------------------------------------------------ MutualInformation gradients
def _grad_close(got, ref, rtol=2e-4):
    """gradients are compared relative to the largest reference entry (they span many decades)."""
    got, ref = got.detach().cpu().double().numpy(), ref.detach().double().numpy()
    scale = np.abs(ref).max()
    assert scale > 0
    np.testing.assert_allclose(got / scale, ref / scale, rtol=0, atol=rtol)


@pytest.mark.parametrize('nb,clip', [(16, None), (11, (0.1, 0.85)), (32, None)])
def test_mi_channelwise_gradient_vs_torch_autograd(ne, nb, clip):
    rng = np.random.default_rng(100 + nb)
    x = rng.uniform(0, 1, (2, 6, 7, 9, 2)).astype(F32)
    y = np.clip(0.6 * x ** 2 + 0.2 + 0.1 * rng.standard_normal(x.shape), 0, 1).astype(F32)
    w = rng.standard_normal((2, 2))
    kw = dict(nb_bins=nb)
    tkw = dict(nb_bins=nb)
    if clip:
        kw.update(min_clip=clip[0], max_clip=clip[1])
        tkw.update(min_clip=clip[0], max_clip=clip[1])
    xg, yg = dev(x).requires_grad_(True), dev(y).requires_grad_(True)
    m = ne.metrics.MutualInformation(**kw)
    out = m.channelwise(xg, yg)
    (out * dev(w.astype(F32))).sum().backward()
    xt, yt = torch.from_numpy(x).double().requires_grad_(True), torch.from_numpy(y).double().requires_grad_(True)
    ref = omi.torch_channelwise(xt, yt, alpha=float(m.soft_bin_alpha), **tkw)
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref.detach().numpy(), **MI_TOL)
    (ref * torch.from_numpy(w)).sum().backward()
    _grad_close(xg.grad, xt.grad)
    _grad_close(yg.grad, yt.grad)
    # the extremal voxels carry the bin-centre path: they must agree too (largest |grad| is often there)
    for gpu, cpu, src in ((xg.grad, xt.grad, x), (yg.grad, yt.grad, y)):
        for idx in (np.argmin(src), np.argmax(src)):
            a, b = float(gpu.flatten()[idx]), float(cpu.flatten()[idx])
            assert abs(a - b) <= 2e-4 * float(cpu.abs().max()) + 1e-9


def test_mi_volumes_explicit_centers_and_one_sided_gradient(ne):
    rng = np.random.default_rng(7)
    x = rng.uniform(0, 1, (3, 400, 1)).astype(F32)
    y = np.clip(x + 0.2 * rng.standard_normal(x.shape), 0, 1).astype(F32)
    centers = np.linspace(0, 1, 12).astype(F32)
    m = ne.metrics.MutualInformation(bin_centers=centers, soft_bin_alpha=40.0)
    xg = dev(x).requires_grad_(True)
    m.volumes(xg, dev(y)).sum().backward()                     # only x needs a gradient
    xt = torch.from_numpy(x).double().requires_grad_(True)
    omi.torch_channelwise(xt, torch.from_numpy(y).double(), nb_bins=None, alpha=40.0, bin_centers=centers).sum().backward()
    _grad_close(xg.grad, xt.grad)


def test_mi_segs_and_volume_seg_gradient(ne):
    rng = np.random.default_rng(8)
    L = 16
    lx = rng.standard_normal((2, 5, 6, 7, L)).astype(F32)
    px = (np.exp(lx) / np.exp(lx).sum(-1, keepdims=True)).astype(F32)
    py = (0.5 * np.roll(px, 1, -1) + 0.5 * px).astype(F32)
    w = torch.tensor([0.7, -1.3])
    a, b = dev(px).requires_grad_(True), dev(py).requires_grad_(True)
    (ne.metrics.MutualInformation().segs(a, b) * w.cuda().float()).sum().backward()
    at, bt = torch.from_numpy(px).double().requires_grad_(True), torch.from_numpy(py).double().requires_grad_(True)
    (omi.torch_maps(at, bt) * w.double()).sum().backward()
    _grad_close(a.grad, at.grad)
    _grad_close(b.grad, bt.grad)
    vol = rng.uniform(0, 1, (2, 5, 6, 7, 1)).astype(F32)
    m = ne.metrics.MutualInformation(nb_bins=L)
    for order in (0, 1):
        v, s = dev(vol).requires_grad_(True), dev(px).requires_grad_(True)
        out = m.volume_seg(v, s) if order == 0 else m.volume_seg(s, v)
        (out * w.cuda().float()).sum().backward()
        vt, st = torch.from_numpy(vol).double().requires_grad_(True), torch.from_numpy(px).double().requires_grad_(True)
        (omi.torch_volume_seg(vt, st, nb_bins=L, alpha=float(m.soft_bin_alpha)) * w.double()).sum().backward()
        _grad_close(v.grad, vt.grad)
        _grad_close(s.grad, st.grad)


@pytest.mark.parametrize('nb', [16, 32])
def test_mi_volumes_gradient_many_ctas(ne, nb):
    """V = 2^17 + 13 voxels per item: the centre-gradient partials of many CTAs of mi_bwd_voxel_kernel are combined
    by mi_bwd_combine_kernel."""
    rng = np.random.default_rng(200 + nb)
    x = rng.uniform(0, 1, (2, 2 ** 17 + 13, 1)).astype(F32)
    y = np.clip(0.5 * x ** 2 + 0.3 + 0.1 * rng.standard_normal(x.shape), 0, 1).astype(F32)
    w = rng.standard_normal(2)
    xg, yg = dev(x).requires_grad_(True), dev(y).requires_grad_(True)
    m = ne.metrics.MutualInformation(nb_bins=nb)
    (m.volumes(xg, yg) * dev(w.astype(F32))).sum().backward()
    xt, yt = torch.from_numpy(x).double().requires_grad_(True), torch.from_numpy(y).double().requires_grad_(True)
    (omi.torch_channelwise(xt, yt, nb_bins=nb, alpha=float(m.soft_bin_alpha)) * torch.from_numpy(w)[:, None]).sum().backward()
    _grad_close(xg.grad, xt.grad)
    _grad_close(yg.grad, yt.grad)
