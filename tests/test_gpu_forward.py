"""
Every forward reduction and convolution kernel path against an fp64 reference, element by element.

Dice, CCE, LocallyConnected3D, the MutualInformation joint histogram and the separable convolution are compared
with the fp64 graphs of oracle/grad.py, oracle/mi.py and oracle/forward.py within the bound of
oracle.forward.value_close:  |got - ref| <= 4 k 2^-24 scale + approx.  scale is the sum of the absolute terms of
the element, k the fp32 rounding depth the kernel's launch geometry gives it, approx the documented error of an
approximate function (named in oracle/forward.py).  Each case names the kernel it is meant to reach;
test_forward_dispatch_launches_each_kernel checks that it does.
"""
import ctypes
import re

import numpy as np
import pytest
import torch

from oracle import forward as of, grad as og

pytestmark = pytest.mark.gpu
MI_TOL = dict(rtol=1e-5, atol=2e-6)


@pytest.fixture(scope='module')
def ne(cuda):
    import neurite_b200
    return neurite_b200


def _g(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# =======================================================================================
# Dice
# =======================================================================================
def _dice_inputs(g, B, S, L, absent=True):
    """one-hot y_true and softmax y_pred; with `absent`, label L-1 appears in neither (0/0 -> 0)."""
    lab = torch.randint(0, max(L - 1, 1) if absent else L, (B,) + S, generator=g, device='cuda')
    t = torch.nn.functional.one_hot(lab, L).float()
    p = torch.softmax(torch.randn((B,) + S + (L,), generator=g, device='cuda'), -1)
    if absent and L > 1:
        p[..., L - 1] = 0
    return t, p


def _dice_check(ne, t, p, laplace, normalize, tag, aligned=True):
    B, L = t.shape[0], t.shape[-1]
    V = t.numel() // (B * L)
    sums, flag = ne.metrics.dice_sums(t, p, normalize=normalize)
    assert int(flag) == 0
    ref = of.torch_dice_sums(t.double(), p.double(), normalize)
    k = of.dice_sums_depth(B, V, L, normalize, aligned)
    of.value_close(sums, ref, ref, k, what='%s dice sums' % tag)          # non-negative terms: scale = value
    d = ne.metrics.Dice(laplace_smoothing=laplace, normalize=normalize).dice(t, p)
    dref = of.torch_dice_fwd(t.double(), p.double(), laplace, normalize)
    # 2 top / bot: the relative errors of top and bot, and the finalize's add and divide
    of.value_close(d, dref, dref, 2 * k + 3, what='%s dice' % tag)
    if laplace == 0 and L > 1:
        assert bool((d[:, L - 1] == 0).all())


@pytest.mark.parametrize('L', [1, 3, 4, 5, 16, 260, 400, 1028])
@pytest.mark.parametrize('laplace', [0.0, 0.1])
@pytest.mark.parametrize('normalize', [False, True])
def test_dice_vs_fp64_reference(ne, L, laplace, normalize):
    """dice_sums_vec4_kernel (L % 4 == 0: q = 1, 4, 65, 100 -> nthr 200), dice_sums_scalar_kernel (L = 1, 3, 5),
    dice_sums_voxel_kernel (normalize, and L = 1028); dice_combine_kernel (3L <= 1024) and
    dice_combine_serial_kernel (L = 400, 1028); Laplace smoothing; an absent label (0/0 -> 0)."""
    g = _g(L * 4 + int(laplace * 10) + 2 * normalize)
    S = (9, 10, 11) if L < 256 else (5, 6, 7)
    t, p = _dice_inputs(g, 2, S, L)
    if normalize:
        t, p = t * 3.0, p * 0.5                                  # the renormalisation has something to do
        t[0, 0, 0, 0] = 0                                        # an all-zero voxel: divide_no_nan
        p[0, 0, 0, 0] = 0
    _dice_check(ne, t, p, laplace, normalize, 'L=%d' % L)


def test_dice_misaligned_operands_take_the_scalar_kernel(ne):
    g = _g(161)
    t, p = _dice_inputs(g, 3, (7, 8, 9), 16)
    bt, bp = torch.empty(t.numel() + 1, device='cuda'), torch.empty(p.numel() + 1, device='cuda')
    tv, pv = bt[1:].view(t.shape), bp[1:].view(p.shape)
    tv.copy_(t)
    pv.copy_(p)
    _dice_check(ne, tv, pv, 0.0, False, 'offset view', aligned=False)


def _abi_dice_sums(ne, t, p, B, V, L, v0, nv, normalize):
    lib = ne._lib.lib
    sums = torch.empty((B, L, 3), device='cuda')
    flag = torch.zeros(1, dtype=torch.int32, device='cuda')
    wsb = lib.nrt_dice_workspace_bytes(B, L)
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    ne._lib.check(lib.nrt_dice_sums_f32(ne._lib.ptr(t), ne._lib.ptr(p), B, V, L, v0, nv, int(normalize), 1,
                                        ne._lib.ptr(sums), ne._lib.ptr(flag), ne._lib.ptr(ws), wsb, _stream()))
    assert int(flag) == 0
    return sums


@pytest.mark.parametrize('L,normalize,kernel', [(16, False, 'vec4'), (5, False, 'scalar'), (5, True, 'voxel'),
                                                 (12, True, 'voxel')])
def test_dice_sums_voxel_range_through_the_abi(ne, L, normalize, kernel):
    """nrt_dice_sums_f32 with v0 > 0: the sums over voxels [v0, v0 + nv) equal those of that slice, for each
    float sums kernel; and nrt_dice_label_sums_i32 over the same range gives the exact counts of the slice."""
    g = _g(L + 100 * normalize)
    B, V = 3, 9001
    t, p = _dice_inputs(g, B, (V,), L, absent=False)
    for v0, nv in ((137, 6001), (V - 1, 1), (0, 4097), (4096, V - 4096), (50, 0)):
        got = _abi_dice_sums(ne, t, p, B, V, L, v0, nv, normalize)
        ts, ps = t[:, v0:v0 + nv], p[:, v0:v0 + nv]
        ref = of.torch_dice_sums(ts.double(), ps.double(), normalize)
        k = of.dice_sums_depth(B, nv, L, normalize)
        of.value_close(got, ref, ref, k, what='%s [%d, %d)' % (kernel, v0, v0 + nv))
    lab_t = torch.randint(-1, L + 1, (B, V), generator=g, device='cuda', dtype=torch.int32)
    lab_p = torch.where(torch.rand((B, V), generator=g, device='cuda') < 0.5, lab_t,
                        torch.randint(-1, L + 1, (B, V), generator=g, device='cuda', dtype=torch.int32))
    lib = ne._lib.lib
    for v0, nv in ((137, 6001), (V - 1, 1), (4096, V - 4096)):
        sums = torch.empty((B, L, 3), device='cuda')
        wsb = lib.nrt_dice_workspace_bytes(B, L)
        ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
        ne._lib.check(lib.nrt_dice_label_sums_i32(ne._lib.ptr(lab_t), ne._lib.ptr(lab_p), B, V, L, v0, nv,
                                                  ne._lib.ptr(sums), ne._lib.ptr(ws), wsb, _stream()))
        ref = of.hard_dice_counts(lab_t[:, v0:v0 + nv], lab_p[:, v0:v0 + nv], L)
        assert torch.equal(sums.long(), ref), (v0, nv)


def test_hard_dice_counts_and_argmax_ties(ne):
    """dice_label_counts_kernel (labels outside [0, L) count nowhere) and argmax_kernel: ties go to the first
    index (tf.argmax); hard Dice from probabilities is the Dice of the two argmax maps, exactly."""
    g = _g(7)
    L = 6
    B, S = 2, (11, 12, 13)
    lt = torch.randint(-2, L + 2, (B,) + S, generator=g, device='cuda')
    lp = torch.where(torch.rand(lt.shape, generator=g, device='cuda') < 0.6, lt,
                     torch.randint(0, L, lt.shape, generator=g, device='cuda'))
    d = ne.metrics.HardDice(nb_labels=L).dice(lt, lp)
    c = of.hard_dice_counts(lt, lp, L).double()
    top, bot = 2 * c[..., 0], c[..., 1] + c[..., 2]
    ref = torch.where(bot != 0, top / torch.where(bot != 0, bot, torch.ones_like(bot)), torch.zeros_like(top))
    assert torch.equal(d, ref.float())                                    # exact counts, one rounding each
    # probabilities with ties: values on a 4-level grid, so many voxels have two or more equal maxima
    x = torch.randint(0, 4, (B,) + S + (L,), generator=g, device='cuda').float() / 4
    x[0, 0, 0, 0] = 0.75
    x[0, 0, 0, 0, L - 1] = 0.75
    idx = ne.metrics.argmax_labels(x)
    assert torch.equal(idx.long(), torch.argmax(x, -1))
    assert int(idx[0, 0, 0, 0]) == 0
    assert int((x == x.max(-1, keepdim=True).values).sum(-1).gt(1).sum()) > 100
    y = torch.softmax(torch.randn(x.shape, generator=g, device='cuda'), -1)
    with pytest.warns(UserWarning):
        dp = ne.metrics.Dice(dice_type='hard').dice(x, y)
    assert torch.equal(dp, ne.metrics.HardDice(nb_labels=L).dice(torch.argmax(x, -1), torch.argmax(y, -1)))


@pytest.mark.parametrize('B', [1, 8])
def test_dice_cfg3_size_vs_fp64_reference(ne, B):
    """160x192x224x16, the longest runs: dice_sums_vec4_kernel at batch 8 (816 float4 per thread) and
    dice_sums_voxel_kernel (normalize) at batch 1 and 8 (about 6.5 k and 52 k voxels into one block accumulator)."""
    g = _g(300 + B)
    S, L = (160, 192, 224), 16
    t, p = _dice_inputs(g, B, S, L, absent=False)
    V = t.numel() // (B * L)
    for normalize in (False, True):
        sums, _ = ne.metrics.dice_sums(t, p, normalize=normalize)
        k = of.dice_sums_depth(B, V, L, normalize)
        for b in range(B):                                   # the fp64 reference one item at a time (memory)
            ref = of.torch_dice_sums(t[b:b + 1].double(), p[b:b + 1].double(), normalize)
            of.value_close(sums[b:b + 1], ref, ref, k, what='cfg3 B=%d item %d normalize=%s' % (B, b, normalize))


# =======================================================================================
# categorical cross-entropy
# =======================================================================================
def _cce_inputs(g, rows, C, logits):
    t = torch.nn.functional.one_hot(torch.randint(0, C, rows, generator=g, device='cuda'), C).float()
    if logits:
        return t, torch.randn(rows + (C,), generator=g, device='cuda') * 3
    p = torch.rand(rows + (C,), generator=g, device='cuda') + 0.05
    flat, tf = p.reshape(-1, C), t.reshape(-1, C)
    flat[0] = 0
    flat[0, 0] = 1                                           # one-hot p: every entry clipped, both ends
    flat[3, 1] = 0                                           # p = 0: that entry clipped at eps
    flat[5, :max(C // 2, 1)] = 0
    tf[5] = 0
    tf[5, 0] = 1                                             # the true label of row 5 is clipped
    return t, p


def _vec4(C, *tensors):
    return C % 4 == 0 and (C // 4) & (C // 4 - 1) == 0 and C // 4 <= 32 and all(
        x is None or x.data_ptr() % 16 == 0 for x in tensors)


def _cce_check(ne, t, p, lw, sw, kw, tag):
    C = p.shape[-1]
    n = p.numel() // C
    vec4 = _vec4(C, t, p, lw)
    args = (t.double(), p.double(), None if lw is None else lw.double(), None if sw is None else sw.double())
    rows_ref = og.torch_cce(*args, reduction='none', **kw)
    scale, k, approx = of.cce_row_bounds(*args, vec4=vec4, **kw)
    for red in ('none', 'sum', 'sum_over_batch_size'):
        out = ne.losses.CategoricalCrossentropy(label_weights=lw, reduction=red, **kw)(t, p, sample_weight=sw)
        if red == 'none':
            of.value_close(out, rows_ref, scale, k, approx, what='%s cce none' % tag)
        else:
            ref = og.torch_cce(*args, reduction=red, **kw)
            s, kk, a = of.cce_reduction_bound(scale, k, approx, rows_ref, n, C, vec4, red)
            of.value_close(out.reshape(()), ref, s, kk, a, what='%s cce %s' % (tag, red))


CCE_VARIANTS = {'plain': dict(), 'weights': dict(), 'smoothing': dict(label_smoothing=0.1),
                'from_logits': dict(from_logits=True)}


@pytest.mark.parametrize('C', [4, 8, 16, 32, 64, 128, 3, 5, 12])
@pytest.mark.parametrize('variant', list(CCE_VARIANTS))
def test_cce_forward_vs_fp64_reference(ne, C, variant):
    """cce_vec4u_kernel<Q> for Q = C/4 in {1, 2, 4, 8, 16, 32} and cce_row_kernel (C = 3, 5, 12, and from_logits
    at any C goes through the same dispatch), every reduction; rows clipped at both ends; label and sample
    weights; 1309 rows (not a multiple of any rows-per-pass)."""
    g = _g(C * 13 + len(variant))
    kw = CCE_VARIANTS[variant]
    rows = (7, 11, 17)
    t, p = _cce_inputs(g, rows, C, kw.get('from_logits', False))
    lw = sw = None
    if variant == 'weights':
        lw = torch.rand(C, generator=g, device='cuda') + 0.5
        sw = torch.rand(rows, generator=g, device='cuda') + 0.5
    _cce_check(ne, t, p, lw, sw, kw, 'C=%d %s' % (C, variant))


def _confident_rows(g, n, C, p_true, exact):
    """n rows whose true class has probability p_true.  exact: p_true = 1 - 2^-j and the rest on one other class
    (the row sum is exactly 1: the kernels' normalisation is exact and only the log is left); else a softmax whose
    true class reaches p_true (the normalisation rounds)."""
    lab = torch.randint(0, C, (n,), generator=g, device='cuda')
    t = torch.nn.functional.one_hot(lab, C).float()
    if exact:
        r = float(np.float32(1 - p_true))
        j = int(np.round(-np.log2(r)))
        p = torch.zeros((n, C), device='cuda')
        p.scatter_(1, lab[:, None], 1 - 2.0 ** -j)
        p.scatter_(1, ((lab + 1) % C)[:, None], 2.0 ** -j)
        return t, p
    z = torch.randn((n, C), generator=g, device='cuda')
    margin = float(np.log(p_true / (1 - p_true) * (C - 1)))
    z.scatter_(1, lab[:, None], margin)
    return t, torch.softmax(z, -1)


@pytest.mark.parametrize('C', [4, 16, 5])
@pytest.mark.parametrize('p_true', [0.9, 0.999, 0.99999, 1 - 1e-7])
def test_cce_confident_rows_vs_fp64_reference(ne, C, p_true):
    """A trained segmentation network's regime: p_true near 1, loss terms down to 1e-7.  Exactly normalised rows
    isolate the log (the float4 kernel, C = 4 and 16; the row kernel, C = 5); softmax rows add the normalisation."""
    g = _g(C * 1000 + int(-np.log10(1 - p_true)))
    for exact in (True, False):
        if exact and p_true == 0.9:
            continue
        t, p = _confident_rows(g, 2003, C, p_true if not exact else 1 - 2.0 ** round(np.log2(1 - p_true)), exact)
        _cce_check(ne, t, p, None, None, {}, 'C=%d p_true=%g exact=%s' % (C, p_true, exact))
        _cce_check(ne, t, p, torch.linspace(0.5, 2, C, device='cuda'), None, {'label_smoothing': 0.01},
                   'C=%d p_true=%g exact=%s smoothing' % (C, p_true, exact))


def test_cce_confident_cfg3_volume_vs_fp64_reference(ne):
    """One 160x192x224x16 volume whose softmax is 0.999-confident, per voxel and summed."""
    g = _g(3)
    n, C = 160 * 192 * 224, 16
    t, p = _confident_rows(g, n, C, 0.999, False)
    _cce_check(ne, t.reshape(1, 160, 192, 224, C), p.reshape(1, 160, 192, 224, C), None, None, {}, 'cfg3 confident')


# =======================================================================================
# LocallyConnected3D
# =======================================================================================
# (name, B, Cin, Cout, kernel size, strides, format, activation, bias, input shape)
LC3D_CASES = [
    ('patch11', 1, 4, 16, (3, 3, 3), (1, 1, 1), 'channels_last', 'relu', True, (6, 7, 8)),
    ('patch12', 2, 4, 8, (2, 3, 2), (2, 1, 2), 'channels_last', None, True, (7, 7, 9)),
    ('patch22', 4, 16, 32, (3, 3, 3), (1, 1, 1), 'channels_last', 'tanh', True, (5, 6, 7)),
    ('patch22-12-11', 7, 16, 16, (3, 3, 3), (1, 1, 1), 'channels_last', 'sigmoid', True, (5, 6, 7)),
    ('rows42', 8, 4, 16, (3, 3, 3), (1, 1, 1), 'channels_last', 'sigmoid', True, (6, 7, 8)),
    ('rows42-patch12-11', 11, 8, 16, (2, 3, 2), (2, 1, 2), 'channels_last', None, False, (7, 7, 9)),
    ('patch24', 8, 4, 8, (3, 3, 3), (1, 1, 1), 'channels_last', 'relu', True, (6, 7, 8)),
    ('stream11', 1, 3, 4, (3, 3, 3), (1, 1, 1), 'channels_last', 'tanh', True, (6, 7, 8)),
    ('stream21', 2, 4, 16, (3, 3, 3), (1, 1, 1), 'channels_first', None, True, (6, 7, 8)),
    ('stream22-11', 5, 3, 32, (2, 3, 2), (2, 1, 2), 'channels_last', 'relu', True, (7, 7, 9)),
    ('stream42-22-11', 13, 1, 8, (3, 3, 3), (1, 1, 1), 'channels_last', 'sigmoid', True, (6, 7, 8)),
    ('stream42-21', 10, 4, 4, (3, 2, 3), (1, 2, 1), 'channels_first', 'tanh', True, (6, 7, 8)),
    ('stream21-64', 3, 16, 64, (3, 3, 3), (1, 1, 1), 'channels_last', None, True, (5, 6, 7)),
    ('generic-128', 2, 16, 128, (3, 3, 3), (1, 1, 1), 'channels_last', 'relu', True, (5, 6, 7)),
    ('generic-3', 3, 4, 3, (3, 3, 3), (1, 1, 1), 'channels_last', 'tanh', True, (6, 7, 8)),
]


def _lc3d_setup(g, B, Cin, Cout, ks, st, fmt, I, bias=True):
    shape = (B, Cin) + I if fmt == 'channels_first' else (B,) + I + (Cin,)
    x = torch.randn(shape, generator=g, device='cuda')
    O = [(I[d] - ks[d]) // st[d] + 1 for d in range(3)]
    P, F = int(np.prod(O)), int(np.prod(ks)) * Cin
    k = torch.randn((P, F, Cout), generator=g, device='cuda') * 0.3
    b = torch.randn(tuple(O) + (Cout,), generator=g, device='cuda') if bias else None
    return x, k, b, O


def _lc3d_check(ne, x, k, b, ks, st, fmt, act, O, tag):
    out = ne.layers.local_conv3d(x, k, b, ks, st, O, fmt, act)
    ref, scale, kk, approx = of.lc3d_fwd_bounds(x, k, b, ks, st, fmt, act)
    of.value_close(out, ref, scale, kk, approx, what='lc3d %s' % tag)


@pytest.mark.parametrize('name,B,Cin,Cout,ks,st,fmt,act,bias,I', LC3D_CASES, ids=[c[0] for c in LC3D_CASES])
def test_lc3d_forward_vs_fp64_reference(ne, name, B, Cin, Cout, ks, st, fmt, act, bias, I):
    """Every kernel of the nrt_lc3d_fwd_f32 dispatch and the batch passes that reach it (the name lists the
    passes): lc3d_patch_kernel <1,1> <1,2> <2,2> <2,4>, lc3d_rows_kernel<4,2>, lc3d_stream_kernel <1,1> <2,1> <2,2>
    <4,2> (channels_first, Cin % 4 != 0), the generic kernel (Cout = 3; Cout = 128 at 3^3 x 16 does not fit the
    ring); Cout = 64 at 3^3 x 16 leaves two ring stages and one consumer group; strides with a ragged F, bias and
    no bias, every activation."""
    g = _g(sum(map(ord, name)))
    x, k, b, O = _lc3d_setup(g, B, Cin, Cout, ks, st, fmt, I, bias)
    _lc3d_check(ne, x, k, b, ks, st, fmt, act, O, name)


@pytest.mark.parametrize('env', [{'NRT_LC3D_STAGES': '3'}, {'NRT_LC3D_WARPS': '1'}, {'NRT_LC3D_WARPS': '2'},
                                 {'NRT_LC3D_STAGES': '3', 'NRT_LC3D_WARPS': '2'}, {'NRT_LC3D_PATCH': '0'},
                                 {'NRT_LC3D_ROWS': '0'}, {'NRT_LC3D_PATCH1': '0'}],
                         ids=lambda e: '-'.join('%s=%s' % kv for kv in e.items()))
def test_lc3d_ring_settings_vs_fp64_reference(ne, monkeypatch, env):
    """The ring depth and consumer-group switches on the patch (B = 1, 2, 4), rows (B = 8) and stream
    (channels_first B = 4, Cin = 3 B = 2) kernels; NRT_LC3D_PATCH=0 sends batches 4-7 of a channels-last input to
    lc3d_stream_kernel<2,2>."""
    for kv in env.items():
        monkeypatch.setenv(*kv)
    g = _g(len(str(env)))
    for B, Cin, Cout, fmt in ((1, 4, 16, 'channels_last'), (2, 8, 8, 'channels_last'), (4, 4, 32, 'channels_last'),
                              (8, 4, 16, 'channels_last'), (4, 4, 16, 'channels_first'), (2, 3, 8, 'channels_last')):
        x, k, b, O = _lc3d_setup(g, B, Cin, Cout, (3, 3, 3), (1, 1, 1), fmt, (6, 7, 8))
        _lc3d_check(ne, x, k, b, (3, 3, 3), (1, 1, 1), fmt, 'relu', O, '%s B=%d Cout=%d %s' % (env, B, Cout, fmt))


def test_lc3d_position_shards_vs_fp64_reference(ne):
    """p0 / p_count ranges (the kernels index weights, bias and output by the local position n and the input
    by p0 + n) on the patch, rows and stream kernels."""
    g = _g(51)
    for B, Cin, fmt in ((2, 4, 'channels_last'), (8, 4, 'channels_last'), (3, 3, 'channels_last'),
                        (4, 4, 'channels_first')):
        x, k, b, O = _lc3d_setup(g, B, Cin, 16, (2, 3, 2), (2, 1, 2), fmt, (7, 7, 9))
        P = int(np.prod(O))
        for p0, pc in ((0, P // 3), (P // 3, P - P // 3 - 1), (P - 1, 1)):
            bb = None if fmt == 'channels_first' else b.reshape(P, 16)[p0:p0 + pc]
            out = ne.layers.local_conv3d(x, k[p0:p0 + pc].contiguous(), bb, (2, 3, 2), (2, 1, 2), O, fmt, None, p0, pc)
            ref, scale, kk, approx = of.lc3d_fwd_bounds(x, k[p0:p0 + pc], bb, (2, 3, 2), (2, 1, 2), fmt, None, p0, pc)
            of.value_close(out, ref, scale, kk, approx, what='lc3d shard B=%d [%d, %d)' % (B, p0, p0 + pc))


# =======================================================================================
# MutualInformation joint histogram (nrt_mi_hist_f32, called as _MiFn.forward calls it)
# =======================================================================================
def _mi_hist(ne, x, xq, nbx, cx, y, yq, nby, cy, B, C, nv, alpha, lo=-np.inf, hi=np.inf):
    lib, ptr = ne._lib.lib, ne._lib.ptr
    items = B * C
    stats = torch.empty((items, nbx * nby + nbx + nby), device='cuda')
    flag = torch.zeros(1, dtype=torch.int32, device='cuda')
    wsb = lib.nrt_mi_workspace_bytes(items, nbx, nby)
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    ne._lib.check(lib.nrt_mi_hist_f32(ptr(x), nv * x.shape[-1], x.shape[-1], int(xq), nbx, ptr(cx),
                                      ptr(y), nv * y.shape[-1], y.shape[-1], int(yq), nby, ptr(cy),
                                      B, C, nv, float(alpha), float(lo), float(hi), ptr(stats), ptr(flag),
                                      ptr(ws), wsb, _stream()))
    mi = torch.empty(items, device='cuda')
    ne._lib.check(lib.nrt_mi_finalize_f32(ptr(stats), items, nbx, nby, 1e-7, ptr(mi), _stream()))
    return stats, mi


def _mi_operand(g, kind, B, nv, C, nb, base=None):
    """'q': intensities [B, nv, C] in [0, 1]; 'm': a probability map [B, nv, nb] (rows sum to 1)."""
    if kind == 'q':
        if base is None:
            return torch.rand((B, nv, C), generator=g, device='cuda')
        return (0.6 * base ** 2 + 0.2 + 0.1 * torch.rand(base.shape, generator=g, device='cuda')).clamp(0, 1)
    z = torch.randn((B, nv, nb), generator=g, device='cuda') * 2
    return torch.softmax(z, -1)


def _mi_spc(nbx, nby):
    """8-voxel MMA steps per chunk of the instantiation launch_mma picks."""
    return 2 if max(nbx, nby) > 16 else 4


def _mi_case(ne, x, xq, nbx, y, yq, nby, B, C, nv, alpha=None, lo=-np.inf, hi=np.inf, centers=None, generic=False,
             per_sm=None, tag=''):
    """Run the ABI on x, y; check every stats element and the MI against the fp64 reference."""
    if alpha is None:
        alpha = float(ne.metrics.MutualInformation(nb_bins=max(nbx if xq else nby, 2)).soft_bin_alpha)

    def cen(v, q, nb):
        if not q:
            return None, None
        c = centers if centers is not None else of.mi_centers_f32(v.cpu().numpy(), nb)
        return torch.from_numpy(np.asarray(c, np.float32)).cuda(), c
    cxd, cxh = cen(x, xq, nbx)
    cyd, cyh = cen(y, yq, nby)
    if xq and centers is None:                               # mi_centers_kernel forms them the same way
        mm = ne.utils.minmax(x)
        assert torch.equal(ne.utils.bin_centers_from_range(mm, nbx), cxd)
    stats, mi = _mi_hist(ne, x, xq, nbx, cxd, y, yq, nby, cyd, B, C, nv, alpha, lo, hi)

    def w(v, q, c, nb):                                      # [B*C, nv, nb]
        vv = v.permute(0, 2, 1).reshape(B * C, nv) if q else v.reshape(B, nv, nb)
        return of.mi_weights(vv, q, c, alpha, lo, hi)
    wx, ex = w(x, xq, cxh, nbx)
    wy, ey = w(y, yq, cyh, nby)
    tc = not generic and nbx <= 32 and nby <= 32
    ref, approx = of.mi_hist_reference(wx, ex, wy, ey, tc)
    kh, km = of.mi_hist_depth(nv, B * C, nbx, nby, not tc, _mi_spc(nbx, nby), per_sm=per_sm)
    npair = nbx * nby
    k = torch.full((stats.shape[1],), float(km), device='cuda')
    k[:npair] = kh
    of.value_close(stats, ref, ref, k, approx, what='mi stats %s' % tag)
    if nv > 0:
        np.testing.assert_allclose(mi.cpu().numpy(), of.mi_from_stats(ref, nbx, nby).cpu().numpy(), **MI_TOL,
                                   err_msg='mi %s' % tag)
    return stats, mi


# (name, x kind, nbx, y kind, nby, channels, env)
MI_CASES = [
    ('mma12-qq-v0', 'q', 16, 'q', 16, 1, {}),
    ('mma12-qq-v2', 'q', 11, 'q', 11, 1, {}),
    ('mma12-qq-c3', 'q', 16, 'q', 16, 3, {}),
    ('mma24-qq', 'q', 32, 'q', 32, 1, {}),
    ('mma12-qm', 'q', 16, 'm', 16, 1, {}),
    ('mma24-qm', 'q', 24, 'm', 24, 1, {}),
    ('mma12-mm', 'm', 16, 'm', 16, 1, {}),
    ('mma12-mq-16x5', 'm', 16, 'q', 5, 1, {}),
    ('mma24-mq-32x12', 'm', 32, 'q', 12, 1, {}),
    ('generic-qq-40', 'q', 40, 'q', 40, 1, {}),
    ('generic-qq-env', 'q', 16, 'q', 16, 1, {'NRT_MI_GENERIC': '1'}),
    ('generic-qm-env', 'q', 24, 'm', 24, 1, {'NRT_MI_GENERIC': '1'}),
    ('ctas1', 'q', 16, 'q', 16, 1, {'NRT_MI_CTAS_PER_SM': '1'}),
    ('ctas2', 'q', 32, 'q', 32, 1, {'NRT_MI_CTAS_PER_SM': '2'}),
    ('ctas8', 'q', 16, 'm', 16, 1, {'NRT_MI_CTAS_PER_SM': '8'}),
]


@pytest.mark.parametrize('nv', [1, 127, 128, 129, 2 ** 17 + 13])
@pytest.mark.parametrize('name,xk,nbx,yk,nby,C,env', MI_CASES, ids=[c[0] for c in MI_CASES])
def test_mi_hist_vs_fp64_reference(ne, monkeypatch, name, xk, nbx, yk, nby, C, env, nv):
    """mi_hist_mma_kernel <1,2> and <2,4> for every quantisation combination, including
    the y-only one and nbx != nby (16x5, 32x12) that only the C ABI reaches; mi_hist_generic_kernel (> 32 bins,
    NRT_MI_GENERIC=1); NRT_MI_CTAS_PER_SM 1, 2, 8; voxel counts around the 128-voxel flush and many CTAs."""
    for kv in env.items():
        monkeypatch.setenv(*kv)
    g = _g(sum(map(ord, name)) + nv)
    B = 2
    x = _mi_operand(g, xk, B, nv, C, nbx)
    y = _mi_operand(g, yk, B, nv, C, nby, base=x if (xk == 'q' and yk == 'q') else None)
    per_sm = int(env['NRT_MI_CTAS_PER_SM']) if 'NRT_MI_CTAS_PER_SM' in env else None
    _mi_case(ne, x, xk == 'q', nbx, y, yk == 'q', nby, B, C, nv, generic='NRT_MI_GENERIC' in env or nbx > 32,
             per_sm=per_sm, tag='%s nv=%d' % (name, nv))


def test_mi_clip_constant_volume_and_explicit_centres_vs_fp64_reference(ne):
    """Inputs outside [min_clip, max_clip] (clipped before quantisation), a constant volume (min = max: every
    centre equal), explicit centres with their own alpha."""
    g = _g(17)
    nv = 3001
    x = torch.rand((2, nv, 1), generator=g, device='cuda') * 1.6 - 0.3
    y = (x + 0.2 * torch.randn(x.shape, generator=g, device='cuda')).clamp(-0.5, 1.5)
    for nb in (16, 32, 40):
        alpha = float(ne.metrics.MutualInformation(nb_bins=nb).soft_bin_alpha)
        _mi_case(ne, x, True, nb, y, True, nb, 2, 1, nv, alpha, lo=0.1, hi=0.85,
                 centers=np.linspace(0.1, 0.85, nb).astype(np.float32), generic=nb > 32, tag='clip nb=%d' % nb)
    const = torch.full((2, nv, 1), 0.37, device='cuda')
    _mi_case(ne, const, True, 16, y, True, 16, 2, 1, nv, tag='constant x')
    centers = np.sort(np.random.default_rng(3).uniform(-0.3, 1.3, 13)).astype(np.float32)
    _mi_case(ne, x, True, 13, y, True, 13, 2, 1, nv, alpha=80.0, centers=centers, tag='explicit centres')


def test_mi_full_size_volume_pair_vs_fp64_reference(ne):
    """BASELINE.json's 160x192x224 volume pair, batch 2, 16 bins: every stats element and the MI against the fp64
    reference; the public volumes() path gives the same MI."""
    g = _g(160)
    nv = 160 * 192 * 224
    x = torch.rand((2, nv, 1), generator=g, device='cuda')
    y = (0.7 * x ** 2 + 0.1 + 0.1 * torch.rand(x.shape, generator=g, device='cuda')).clamp(0, 1)
    _, mi = _mi_case(ne, x, True, 16, y, True, 16, 2, 1, nv, tag='160x192x224')
    m = ne.metrics.MutualInformation(nb_bins=16)
    assert torch.equal(m.volumes(x.reshape(2, 160, 192, 224, 1), y.reshape(2, 160, 192, 224, 1)), mi)


# =======================================================================================
# separable convolution (nrt_sepconv_axis_f32)
# =======================================================================================
# (name, shape [B, *space, C], axis, K, padding, stride, dilation, env)
CONV_CASES = [
    ('col4_64', (2, 70, 12, 40, 1), 0, 7, 'SAME', 1, 1, {}),
    ('col4_64-K32', (1, 90, 8, 36, 1), 0, 32, 'SAME', 1, 1, {}),
    ('col-K41', (1, 90, 8, 36, 1), 0, 41, 'SAME', 1, 1, {}),
    ('col4_64-even', (2, 20, 33, 12, 4), 1, 8, 'SAME', 1, 1, {}),
    ('col4_64-valid', (2, 70, 12, 40, 1), 0, 6, 'VALID', 1, 1, {}),
    ('col', (2, 70, 11, 39, 1), 0, 7, 'SAME', 1, 1, {}),
    ('col-even-K40', (1, 90, 8, 36, 1), 0, 40, 'SAME', 1, 1, {}),
    ('col-ragged', (2, 50, 33, 1), 0, 5, 'SAME', 1, 1, {}),
    ('row-inner1', (3, 300, 1), 0, 41, 'SAME', 1, 1, {}),
    ('row-inner1-even', (2, 9, 17, 70, 1), 2, 6, 'SAME', 1, 1, {}),
    ('row-inner2', (2, 40, 2000, 2), 1, 7, 'SAME', 1, 1, {}),
    ('row-inner3', (1, 9, 70, 3), 1, 13, 'SAME', 1, 1, {}),
    ('row-inner17', (2, 130, 17), 0, 4, 'SAME', 1, 1, {}),
    ('generic-stride', (2, 30, 17, 40, 1), 0, 5, 'SAME', 2, 1, {}),
    ('row-dilation', (2, 30, 17, 40, 1), 2, 5, 'SAME', 1, 3, {}),
    ('generic-dilation', (2, 30, 17, 40, 1), 0, 5, 'SAME', 1, 3, {}),
    ('generic-valid-stride', (2, 31, 40, 3), 1, 8, 'VALID', 3, 1, {}),
    ('generic-env', (2, 30, 17, 40, 1), 0, 7, 'SAME', 1, 1, {'NRT_CONV_GENERIC': '1'}),
    ('generic-row-valid', (3, 300, 1), 0, 41, 'VALID', 1, 1, {}),
]


@pytest.mark.parametrize('name,shape,axis,K,padding,stride,dil,env', CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_sepconv_pass_vs_fp64_reference(ne, monkeypatch, name, shape, axis, K, padding, stride, dil, env):
    """sepconv_col4_kernel (K <= 32), sepconv_col_kernel (inner not a multiple of 4, K = 40 and 41 whose 64-row
    float4 tile would not fit 48 KB), sepconv_row_kernel (inner = 1, 2, 3, 17 < 32, and a dilated pass),
    sepconv_generic_kernel (stride, dilation on a column axis, VALID on a row, NRT_CONV_GENERIC=1); K up to 41, even K
    under SAME, VALID; random kernels with cancellation."""
    for kv in env.items():
        monkeypatch.setenv(*kv)
    g = _g(sum(map(ord, name)))
    x = torch.randn(shape, generator=g, device='cuda')
    k = torch.randn(K, generator=g, device='cuda')
    out = ne.utils.separable_conv(x, [k], axis=axis, batched=True, padding=padding, strides=stride, dilations=dil)
    ref = of.torch_separable_conv(x.double(), [k.double()], [axis], padding, [stride], [dil])
    scale, kk = of.sepconv_bounds(x, [k], [axis], padding, [stride], [dil])
    of.value_close(out, ref, scale, kk, what='sepconv %s' % name)


def test_gaussian_blur_passes_vs_fp64_reference(ne):
    """A three-pass blur (column, column, row kernels): the bound chains the passes."""
    g = _g(99)
    x = torch.randn((2, 40, 33, 70, 1), generator=g, device='cuda')
    sigma = [1.3, 2.0, 0.8]
    ks = [k.cuda() for k in ne.utils.gaussian_kernel(sigma, separate=True)]
    out = ne.layers.GaussianBlur(sigma=sigma)(x)
    ref = of.torch_separable_conv(x.double(), [k.double() for k in ks], [0, 1, 2])
    scale, kk = of.sepconv_bounds(x, ks, [0, 1, 2])
    of.value_close(out, ref, scale, kk, what='blur')


# =======================================================================================
# dispatch
# =======================================================================================
def test_forward_dispatch_launches_each_kernel(ne, monkeypatch):
    """The path tests above rely on the dispatch: record which kernels representative cases launch."""
    from torch.profiler import profile, ProfilerActivity

    def names(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [re.sub(r'\s+', '', e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    if not names(lambda: torch.ones(4, device='cuda').add_(1)):
        pytest.skip('torch.profiler recorded no CUDA events on this machine')

    def expect(fn, want, absent=(), env=None):
        for kv in (env or {}).items():
            monkeypatch.setenv(*kv)
        ns = names(fn)
        for kv in (env or {}).items():
            monkeypatch.delenv(kv[0])
        for w in want:
            assert any(w in n for n in ns), (w, ns)
        for a in absent:
            assert not any(a in n for n in ns), (a, ns)
        return ns

    g = _g(5)
    # Dice
    for L, normalize, want, comb in ((16, False, 'dice_sums_vec4_kernel<4>', 'dice_combine_kernel'),
                                     (400, False, 'dice_sums_vec4_kernel<4>', 'dice_combine_serial_kernel'),
                                     (5, False, 'dice_sums_scalar_kernel', 'dice_combine_kernel'),
                                     (5, True, 'dice_sums_voxel_kernel', 'dice_combine_kernel'),
                                     (1028, False, 'dice_sums_voxel_kernel', 'dice_combine_serial_kernel')):
        t, p = _dice_inputs(g, 2, (4, 5, 6), L)
        ns = expect(lambda: ne.metrics.dice_sums(t, p, normalize=normalize), [want, comb])
        if comb == 'dice_combine_kernel':
            assert not any('dice_combine_serial_kernel' in n for n in ns), ns
    lt = torch.randint(0, 4, (2, 9, 9), generator=g, device='cuda')
    expect(lambda: ne.metrics.HardDice(nb_labels=4).dice(lt, lt), ['dice_label_counts_kernel'])
    x = torch.rand((2, 9, 4), generator=g, device='cuda')
    expect(lambda: ne.metrics.argmax_labels(x), ['argmax_kernel'])
    # CCE
    for C in (4, 8, 16, 32, 64, 128):
        t, p = _cce_inputs(g, (3, 50), C, False)
        expect(lambda: ne.losses.CategoricalCrossentropy()(t, p), ['cce_vec4u_kernel<%d,4>' % (C // 4)],
               ['cce_row_kernel'])
    for C in (3, 5, 12):
        t, p = _cce_inputs(g, (3, 50), C, False)
        expect(lambda: ne.losses.CategoricalCrossentropy()(t, p), ['cce_row_kernel'], ['cce_vec4u_kernel'])
    # LocallyConnected3D
    for name, B, Cin, Cout, ks, st, fmt, act, bias, I in LC3D_CASES:
        x, k, b, O = _lc3d_setup(g, B, Cin, Cout, ks, st, fmt, I, bias)
        want = {'patch11': ['lc3d_patch_kernel<1,1>'], 'patch12': ['lc3d_patch_kernel<1,2>'],
                'patch22': ['lc3d_patch_kernel<2,2>'],
                'patch22-12-11': ['lc3d_patch_kernel<2,2>', 'lc3d_patch_kernel<1,2>', 'lc3d_patch_kernel<1,1>'],
                'rows42': ['lc3d_rows_kernel<4,2>'],
                'rows42-patch12-11': ['lc3d_rows_kernel<4,2>', 'lc3d_patch_kernel<1,2>', 'lc3d_patch_kernel<1,1>'],
                'patch24': ['lc3d_patch_kernel<2,4>'], 'stream11': ['lc3d_stream_kernel<1,1>'],
                'stream21': ['lc3d_stream_kernel<2,1>'],
                'stream22-11': ['lc3d_stream_kernel<2,2>', 'lc3d_stream_kernel<1,1>'],
                'stream42-22-11': ['lc3d_stream_kernel<4,2>', 'lc3d_stream_kernel<2,2>', 'lc3d_stream_kernel<1,1>'],
                'stream42-21': ['lc3d_stream_kernel<4,2>', 'lc3d_stream_kernel<2,1>'],
                'stream21-64': ['lc3d_stream_kernel<2,1>', 'lc3d_stream_kernel<1,1>'],
                'generic-128': ['lc3d_generic_kernel'], 'generic-3': ['lc3d_generic_kernel']}[name]
        kinds = ('lc3d_patch_kernel', 'lc3d_rows_kernel', 'lc3d_stream_kernel', 'lc3d_generic_kernel')
        ns = expect(lambda: ne.layers.local_conv3d(x, k, b, ks, st, O, fmt, act), want)
        got = sorted({re.search(r'(lc3d_\w+_kernel(<\d,\d>)?)', n).group(1) for n in ns if any(s in n for s in kinds)})
        assert got == sorted(set(want)), (name, got)
    x, k, b, O = _lc3d_setup(g, 5, 4, 16, (3, 3, 3), (1, 1, 1), 'channels_last', (6, 7, 8))
    expect(lambda: ne.layers.local_conv3d(x, k, b, (3, 3, 3), (1, 1, 1), O), ['lc3d_stream_kernel<2,2>'],
           ['lc3d_patch_kernel'], env={'NRT_LC3D_PATCH': '0'})
    # MI
    for name, xk, nbx, yk, nby, C, env in MI_CASES:
        xx = _mi_operand(g, xk, 2, 300, C, nbx)
        yy = _mi_operand(g, yk, 2, 300, C, nby, base=xx if (xk == 'q' and yk == 'q') else None)
        cx = torch.linspace(0, 1, nbx, device='cuda') if xk == 'q' else None
        cy = torch.linspace(0, 1, nby, device='cuda') if yk == 'q' else None
        generic = 'NRT_MI_GENERIC' in env or nbx > 32
        mt, nt = (1, 2) if max(nbx, nby) <= 16 else (2, 4)
        minb = 2 if xk == yk == 'q' else 1
        want = 'mi_hist_generic_kernel' if generic else 'mi_hist_mma_kernel<%d,%d,%s,%s,%d,%d>' % (
            mt, nt, str(xk == 'q').lower(), str(yk == 'q').lower(), _mi_spc(nbx, nby), minb)
        expect(lambda: _mi_hist(ne, xx, xk == 'q', nbx, cx, yy, yk == 'q', nby, cy, 2, C, 300, 30.0),
               [want, 'mi_combine_kernel'], env=env)
    # separable convolution
    for name, shape, axis, K, padding, stride, dil, env in CONV_CASES:
        x = torch.randn(shape, generator=g, device='cuda')
        kern = torch.randn(K, generator=g, device='cuda')
        want = {'col4_64': 'sepconv_col4_kernel', 'col': 'sepconv_col_kernel',
                'row': 'sepconv_row_kernel', 'generic': 'sepconv_generic_kernel'}[name.split('-')[0]]
        expect(lambda: ne.utils.separable_conv(x, [kern], axis=axis, batched=True, padding=padding, strides=stride,
                                               dilations=dil), [want], env=env)
