"""
CPU checks of the fp64 forward references (oracle/forward.py): run in fp32 they reproduce the numpy oracle --
within 1e-6 relative for Dice with normalize, the separable convolution and the MI joint histogram, exactly for
hard-Dice counts and the bin centres -- so they are the same graphs.  And an fp32 evaluation of each graph stays
inside the bound value_close puts on the kernels, so the bounds leave room for a legitimate fp32 order.
"""
import numpy as np
import pytest
import torch

from oracle import conv as oconv, forward as of, grad as og, metrics as om, mi as omi
from oracle.interp import tf_linspace_f32

F32 = np.float32
SMS = 132


@pytest.mark.parametrize('L', [1, 4, 5])
@pytest.mark.parametrize('laplace', [0.0, 0.2])
def test_torch_dice_normalize_fp32_is_the_numpy_oracle(L, laplace):
    rng = np.random.default_rng(L)
    t = (np.eye(L, dtype=F32)[rng.integers(0, L, (2, 5, 6))] * 3).astype(F32)
    p = rng.uniform(0, 2, t.shape).astype(F32)
    t[0, 0, 0] = 0
    p[1, 2, 3] = 0
    got = of.torch_dice_fwd(torch.from_numpy(t), torch.from_numpy(p), laplace, normalize=True).numpy()
    ref = om.Dice(laplace_smoothing=laplace, normalize=True).dice(t, p)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)


def test_hard_dice_counts_are_the_numpy_oracle_exactly():
    rng = np.random.default_rng(3)
    L = 5
    t = rng.integers(-1, L + 2, (3, 7, 8))
    p = np.where(rng.uniform(size=t.shape) < 0.5, t, rng.integers(0, L, t.shape))
    c = of.hard_dice_counts(torch.from_numpy(t), torch.from_numpy(p), L).double()
    top, bot = 2 * c[..., 0], c[..., 1] + c[..., 2]
    got = torch.where(bot != 0, top / torch.where(bot != 0, bot, torch.ones_like(bot)), torch.zeros_like(top)).float()
    ref = om.Dice(dice_type='hard', input_type='max_label', nb_labels=L).dice(t, p)
    assert np.array_equal(got.numpy(), ref)


SEP = [((2, 13, 6, 1), 0, 7, 'SAME', 1, 1), ((2, 13, 6, 1), 0, 4, 'SAME', 1, 1), ((2, 13, 6, 3), 1, 4, 'VALID', 1, 1),
       ((1, 17, 5, 2), 0, 5, 'SAME', 2, 1), ((1, 17, 5, 2), 0, 3, 'SAME', 1, 3), ((1, 20, 2), 0, 6, 'VALID', 3, 1),
       ((1, 9, 1), 0, 41, 'SAME', 1, 1)]


@pytest.mark.parametrize('shape,axis,K,padding,stride,dil', SEP)
def test_torch_conv_axis_fp32_is_the_numpy_oracle(shape, axis, K, padding, stride, dil):
    rng = np.random.default_rng(K * 10 + stride)
    x = rng.standard_normal(shape).astype(F32)
    k = rng.standard_normal(K).astype(F32)
    got = of.torch_separable_conv(torch.from_numpy(x), [torch.from_numpy(k)], [axis], padding, [stride], [dil]).numpy()
    ref = oconv.separable_conv(x, [k], axis=axis, batched=True, padding=padding, strides=stride, dilations=dil)
    assert got.shape == ref.shape
    scale = of.torch_separable_conv(torch.from_numpy(np.abs(x)), [torch.from_numpy(np.abs(k))], [axis], padding,
                                    [stride], [dil]).numpy()
    assert np.all(np.abs(got - ref) <= 1e-6 * scale)
    # fp32 evaluation vs fp64 reference within the kernel bound
    r64 = of.torch_separable_conv(torch.from_numpy(x).double(), [torch.from_numpy(k).double()], [axis], padding,
                                  [stride], [dil])
    s, kk = of.sepconv_bounds(torch.from_numpy(x), [torch.from_numpy(k)], [axis], padding, [stride], [dil])
    of.value_close(torch.from_numpy(got), r64, s, kk)


@pytest.mark.parametrize('nb', [1, 2, 7, 16, 33])
def test_mi_centres_are_tf_linspace_of_the_fp32_range(nb):
    rng = np.random.default_rng(nb)
    x = rng.uniform(-3, 5, 1000).astype(F32)
    assert np.array_equal(of.mi_centers_f32(x, nb), tf_linspace_f32(x.min(), x.max(), nb))


@pytest.mark.parametrize('nb', [5, 16])
def test_mi_hist_reference_fp32_is_the_numpy_oracle(nb):
    """The joint histogram and marginals from mi_weights / mi_hist_reference, evaluated in fp32, give the oracle's
    MI within 1e-6 relative, and the fp64 stats sit inside their bound of the fp32 ones."""
    rng = np.random.default_rng(nb)
    x = rng.uniform(0, 1, (2, 500, 1)).astype(F32)
    y = np.clip(0.6 * x * x + 0.2 + 0.1 * rng.standard_normal(x.shape), 0, 1).astype(F32)
    alpha = float(omi.default_alpha(nb))
    cx, cy = of.mi_centers_f32(x, nb), of.mi_centers_f32(y, nb)
    w = []
    for v, c in ((x, cx), (y, cy)):
        xc = torch.from_numpy(v[..., 0])[..., None]
        w.append(torch.exp(-F32(alpha) * (xc - torch.from_numpy(c)) ** 2))
    z = torch.zeros_like(w[0])
    stats32, _ = of.mi_hist_reference(w[0], z, w[1], z, False)
    got = of.mi_from_stats(stats32.double(), nb, nb).numpy()
    np.testing.assert_allclose(got, omi.MutualInformation(nb_bins=nb).volumes(x, y), rtol=1e-6, atol=1e-7)
    wx, ex = of.mi_weights(torch.from_numpy(x[..., 0]), True, cx, alpha, -np.inf, np.inf)
    wy, ey = of.mi_weights(torch.from_numpy(y[..., 0]), True, cy, alpha, -np.inf, np.inf)
    ref, approx = of.mi_hist_reference(wx, ex, wy, ey, False)
    of.value_close(stats32, ref, ref, 500 + 1, approx)


@pytest.mark.parametrize('C', [4, 5, 16])
@pytest.mark.parametrize('kw', [dict(), dict(label_smoothing=0.1), dict(from_logits=True)])
def test_cce_bound_holds_for_an_fp32_evaluation(C, kw):
    """og.torch_cce in fp32 (its own summation order) lies within cce_row_bounds of the fp64 graph, on confident
    rows, exactly normalised rows and rows clipped at both ends."""
    g = torch.Generator().manual_seed(C)
    n = 600
    lab = torch.randint(0, C, (n,), generator=g)
    t = torch.nn.functional.one_hot(lab, C).float()
    if kw.get('from_logits'):
        p = torch.randn((n, C), generator=g) * 4
    else:
        z = torch.randn((n, C), generator=g)
        z[torch.arange(n), lab] += torch.linspace(0, 20, n)
        p = torch.softmax(z, -1)
        p[:50] = 0
        p[:50, 0] = 1
        p[50:100] = 0
        p[50:100, 1] = 1 - 2.0 ** -10
        p[50:100, 2] = 2.0 ** -10
    lw = torch.rand(C, generator=g) + 0.5
    got = og.torch_cce(t, p, lw, reduction='none', **kw)
    ref = og.torch_cce(t.double(), p.double(), lw.double(), reduction='none', **kw)
    scale, k, approx = of.cce_row_bounds(t, p, lw, None, vec4=False, **kw)
    of.value_close(got, ref, scale, k, approx)


def test_lc3d_bound_holds_for_an_fp32_evaluation():
    g = torch.Generator().manual_seed(4)
    for fmt, act in (('channels_last', 'tanh'), ('channels_first', 'sigmoid')):
        x = torch.randn((2, 3, 6, 7, 5) if fmt == 'channels_first' else (2, 6, 7, 5, 3), generator=g)
        k = torch.randn((4 * 5 * 3, 27 * 3, 8), generator=g) * 0.3
        b = torch.randn((4, 5, 3, 8), generator=g)
        pre = og.torch_local_conv3d(x, k, b, (3, 3, 3), (1, 1, 1), fmt)
        got = of.LC3D_ACT[act][0](pre)
        ref, scale, kk, approx = of.lc3d_fwd_bounds(x, k, b, (3, 3, 3), (1, 1, 1), fmt, act)
        of.value_close(got, ref, scale, kk, approx)


def test_depth_helpers_follow_the_host_dispatch():
    """Spot values of the launch-geometry helpers (132 SMs)."""
    # cfg 3 Dice, batch 8: 132 blocks of 208,896 float4 = 816 per thread + a 64-thread fold + the combine
    assert of.dice_blocks(160 * 192 * 224 * 4, 8, SMS) == 132
    assert of.dice_sums_depth(8, 160 * 192 * 224, 16, sms=SMS) == 816 + 64 + 1
    # L = 400: q = 100 -> 200 active threads, fold of 2
    assert of.dice_sums_depth(2, 210, 400, sms=SMS) == 20 + 2 + 1
    assert of.mi_blocks(2 ** 17 + 13, 2, SMS) == 129 and of.mi_blocks(100, 2, SMS) == 1
    assert of.mi_blocks(10 ** 8, 1, SMS, per_sm=8) == 592
    # CCE at batch 4, C = 16: 1056 CTAs of 256 rows per pass, 102 passes of 4 rows
    assert of.cce_rows_per_thread(4 * 160 * 192 * 224, 16, True, SMS) == 4 * 102
