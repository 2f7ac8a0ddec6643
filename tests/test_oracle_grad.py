"""
CPU checks of the gradient oracle (oracle/grad.py): run in fp32, the differentiable torch graphs
reproduce the numpy oracle -- bit for bit for the interpolation graphs, within 1e-6 relative for
Dice, CCE and LocallyConnected3D -- so they are the same graph; in fp64 torch.autograd.gradcheck
passes on each of them away from kinks, so their autograd gradients are that graph's derivative.
"""
import numpy as np
import pytest
import torch

from oracle import grad as og, interp as oi, lc3d as olc, metrics as om

F32 = np.float32


def _planted_loc(rng, S, O, spread):
    """[*O, D] fp32 locations: uniform over the volume +- spread, with exact integers, exact halves, 0, S-1
    and points just outside planted on purpose."""
    D = len(S)
    loc = rng.uniform(-spread, np.array(S) - 1 + spread, tuple(O) + (D,)).astype(F32)
    flat = loc.reshape(-1, D)
    n = flat.shape[0]
    for d in range(D):
        pick = rng.choice(n, size=max(1, n // 6), replace=False)
        kind = rng.integers(0, 5, pick.size)
        vals = np.select([kind == 0, kind == 1, kind == 2, kind == 3],
                         [rng.integers(0, S[d], pick.size), rng.integers(0, S[d], pick.size) + 0.5, 0.0, S[d] - 1.0],
                         S[d] - 0.75)
        flat[pick, d] = vals.astype(F32)
    return loc


@pytest.mark.parametrize('D,C', [(1, 1), (2, 3), (3, 1), (3, 4)])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', -1.5), ('nearest', None), ('nearest', 0.5)])
def test_torch_interpn_fp32_is_the_numpy_oracle_bit_for_bit(D, C, method, fill):
    rng = np.random.default_rng(10 * D + C)
    S = [7, 5, 6][:D]
    vol = rng.standard_normal(tuple(S) + (C,)).astype(F32)
    loc = _planted_loc(rng, S, (4, 9), 1.5)
    got = og.torch_interpn(torch.from_numpy(vol), torch.from_numpy(loc), method, fill).numpy()
    assert np.array_equal(got, oi.interpn(vol, loc, method, fill))


@pytest.mark.parametrize('shape,C', [((6, 7, 8), 1), ((5, 6, 9), 3), ((9, 10), 2), ((17,), 1)])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', 0.5), ('nearest', None)])
def test_torch_warp_fp32_is_the_numpy_oracle_bit_for_bit(shape, C, method, fill):
    rng = np.random.default_rng(len(shape) + C)
    vol = rng.standard_normal((2,) + shape + (C,)).astype(F32)
    flow = rng.uniform(-3, 3, (2,) + shape + (len(shape),)).astype(F32)
    flow[..., 0].reshape(-1)[::5] = 0.5                      # exact halves and integers in the sum coord + flow
    flow[..., -1].reshape(-1)[::7] = -2.0
    got = og.torch_warp(torch.from_numpy(vol), torch.from_numpy(flow), method, fill).numpy()
    assert np.array_equal(got, oi.spatial_transformer(vol, flow, method, fill_value=fill))


@pytest.mark.parametrize('shape,zoom', [((5, 6, 7), [2, 1.5, 0.8]), ((3, 8), [1.7, 0.5]), ((3,), 1.7),
                                        ((4, 5, 3), [0.3, 0.5, 3.7])])
@pytest.mark.parametrize('method', ['linear', 'nearest'])
def test_torch_resize_fp32_is_the_numpy_oracle_bit_for_bit(shape, zoom, method):
    rng = np.random.default_rng(len(shape))
    x = rng.standard_normal((2,) + shape + (3,)).astype(F32)
    got = og.torch_resize(torch.from_numpy(x), zoom, method).numpy()
    assert np.array_equal(got, oi.resize_layer(x, zoom, method))


def test_torch_vec_int_fp32_is_the_numpy_oracle_bit_for_bit():
    rng = np.random.default_rng(3)
    vel = rng.uniform(-6, 6, (2, 7, 8, 9, 3)).astype(F32)
    assert np.array_equal(og.torch_vec_int(torch.from_numpy(vel), 5).numpy(), oi.vec_int(vel, 5))
    vel2 = rng.uniform(-4, 4, (1, 11, 12, 2)).astype(F32)
    assert np.array_equal(og.torch_vec_int(torch.from_numpy(vel2), 4).numpy(), oi.vec_int(vel2, 4))


@pytest.mark.parametrize('laplace', [0.0, 0.1])
def test_torch_dice_matches_the_numpy_oracle(laplace):
    rng = np.random.default_rng(4)
    L = 5
    t = np.eye(L, dtype=F32)[rng.integers(0, 4, (3, 6, 7, 8))]       # label 4 absent
    p = rng.uniform(0, 1, t.shape).astype(F32)
    p[..., 4] = 0
    p /= p.sum(-1, keepdims=True)
    got = og.torch_dice(torch.from_numpy(t), torch.from_numpy(p), laplace).numpy()
    ref = om.Dice(laplace_smoothing=laplace).dice(t, p)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)


@pytest.mark.parametrize('kw', [dict(), dict(from_logits=True), dict(label_smoothing=0.1), dict(reduction='sum'),
                                dict(reduction='none'), dict(label_smoothing=0.2, from_logits=True, reduction='none')])
@pytest.mark.parametrize('weights', [False, True])
def test_torch_cce_matches_the_numpy_oracle(kw, weights):
    rng = np.random.default_rng(5)
    C = 6
    t = np.eye(C, dtype=F32)[rng.integers(0, C, (2, 5, 6))]
    p = (rng.uniform(0, 1, t.shape) + 0.05).astype(F32)
    p[0, 0, 0] = [1, 0, 0, 0, 0, 0]                                    # clipped entries
    lw = (rng.uniform(0, 1, C) + 0.5).astype(F32) if weights else None
    sw = (rng.uniform(0, 1, (2, 5, 6)) + 0.5).astype(F32) if weights else None
    got = og.torch_cce(torch.from_numpy(t), torch.from_numpy(p), None if lw is None else torch.from_numpy(lw),
                       None if sw is None else torch.from_numpy(sw), **kw).numpy()
    ref = om.categorical_crossentropy(t, p, label_weights=lw, sample_weight=sw, **kw)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)


@pytest.mark.parametrize('fmt', ['channels_last', 'channels_first'])
@pytest.mark.parametrize('ks,st', [((3, 3, 3), (1, 1, 1)), ((2, 3, 2), (2, 1, 2))])
def test_torch_local_conv3d_matches_the_numpy_oracle(fmt, ks, st):
    rng = np.random.default_rng(6)
    B, I, Cin, Cout = 2, (6, 7, 8), 3, 4
    x = rng.standard_normal((B,) + I + (Cin,)).astype(F32)
    if fmt == 'channels_first':
        x = np.ascontiguousarray(np.moveaxis(x, -1, 1))
    O = olc.output_shape(I, ks, st)
    P, F = int(np.prod(O)), int(np.prod(ks)) * Cin
    k = (0.3 * rng.standard_normal((P, F, Cout))).astype(F32)
    b = rng.standard_normal(O + (Cout,)).astype(F32)
    got = og.torch_local_conv3d(torch.from_numpy(x), torch.from_numpy(k), torch.from_numpy(b), ks, st, fmt).numpy()
    ref = olc.locally_connected_3d(x, k, b, ks, st, data_format=fmt)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max())
    # a position range is the matching slice of the whole output
    p0, pc = 5, P - 9
    part = og.torch_local_conv3d(torch.from_numpy(x), torch.from_numpy(k[p0:p0 + pc]), None, ks, st, fmt, p0, pc)
    whole = og.torch_local_conv3d(torch.from_numpy(x), torch.from_numpy(k), None, ks, st, fmt)
    whole = whole.permute(0, 2, 3, 4, 1) if fmt == 'channels_first' else whole
    assert torch.equal(part, whole.reshape(B, P, Cout)[:, p0:p0 + pc])


# ------------------------------------------------------------------ gradchecks (fp64, away from kinks)
def _off_kinks(loc):
    """move locations at least 0.1 away from integers and from the volume edges' kinks"""
    frac = loc - torch.floor(loc)
    return torch.floor(loc) + torch.clamp(frac, 0.1, 0.9)


@pytest.mark.parametrize('D,C,fill', [(1, 2, None), (2, 1, 0.5), (3, 2, None)])
def test_gradcheck_interpn_and_warp(D, C, fill):
    g = torch.Generator().manual_seed(D)
    S = (4, 5, 3)[:D]
    vol = torch.randn(S + (C,), generator=g, dtype=torch.float64, requires_grad=True)
    loc = _off_kinks(torch.rand((3, 2, D), generator=g, dtype=torch.float64) * (torch.tensor(S) + 1) - 1)
    loc.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v, l: og.torch_interpn(v, l, 'linear', fill, False), (vol, loc))
    flow = torch.rand((1,) + S + (D,), generator=g, dtype=torch.float64) * 3 - 1.5
    flow = _off_kinks(og.warp_loc(flow[0]))[None] - og.warp_loc(torch.zeros_like(flow[0]))[None]
    flow = flow.float().double().requires_grad_(True)
    v1 = vol.detach()[None].clone().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v, f: og.torch_warp(v, f, 'linear', fill, False), (v1, flow))


def test_gradcheck_resize_vec_int_dice_cce_lc3d():
    g = torch.Generator().manual_seed(1)
    x = torch.randn((1, 3, 4, 2), generator=g, dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda v: og.torch_resize(v, [1.5, 0.75], 'linear', False), (x,))
    vel = (torch.rand((1, 5, 6, 2), generator=g, dtype=torch.float64) * 1.6 + 0.2).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v: og.torch_vec_int(v, 2, False), (vel,))
    t = torch.rand((2, 3, 4, 3), generator=g, dtype=torch.float64, requires_grad=True)
    p = torch.rand((2, 3, 4, 3), generator=g, dtype=torch.float64, requires_grad=True)
    for lap in (0.0, 0.1):
        assert torch.autograd.gradcheck(lambda a, b: og.torch_dice(a, b, lap), (t, p))
    tt = torch.rand((2, 3, 4), generator=g, dtype=torch.float64)
    pp = (torch.rand((2, 3, 4), generator=g, dtype=torch.float64) + 0.1).requires_grad_(True)
    lw = torch.rand(4, generator=g, dtype=torch.float64) + 0.5
    sw = torch.rand((2, 3), generator=g, dtype=torch.float64) + 0.5
    for kw in (dict(), dict(from_logits=True), dict(label_smoothing=0.1, reduction='none'), dict(reduction='sum')):
        assert torch.autograd.gradcheck(lambda q: og.torch_cce(tt, q, lw, sw, **kw), (pp,))
    for fmt in ('channels_last', 'channels_first'):
        xx = torch.randn((2, 2, 4, 3, 5) if fmt == 'channels_first' else (2, 4, 3, 5, 2), generator=g,
                         dtype=torch.float64, requires_grad=True)
        kk = torch.randn((2 * 2 * 2, 8 * 2, 3), generator=g, dtype=torch.float64, requires_grad=True)
        bb = torch.randn((2, 2, 2, 3), generator=g, dtype=torch.float64, requires_grad=True)
        assert torch.autograd.gradcheck(
            lambda a, k, b: og.torch_local_conv3d(a, k, b, (2, 2, 2), (2, 1, 2), fmt), (xx, kk, bb))


def test_warp_loc_is_the_fp32_sum_with_an_fp64_gradient():
    g = torch.Generator().manual_seed(11)
    flow = (torch.rand((5, 6, 7, 3), generator=g, dtype=torch.float64) * 20 - 10)
    flow[0, 0, 0] = torch.tensor([-1e-9, 1e-9, 0.0], dtype=torch.float64)          # locations at and next to 0
    f = flow.clone().requires_grad_(True)
    loc = og.warp_loc(f)
    assert torch.equal(loc, og.warp_loc(flow.float()).double())
    gout = torch.randn(loc.shape, generator=g, dtype=torch.float64)
    loc.backward(gout)
    assert torch.equal(f.grad, gout)                                                 # not rounded to fp32


def test_grad_close_is_per_element():
    ref = torch.tensor([1.0, 1e-6, 0.0], dtype=torch.float64)
    scale = ref.abs()
    og.grad_close(ref + torch.tensor([1e-7, 1e-13, 0.0], dtype=torch.float64), ref, scale, 1)
    with pytest.raises(AssertionError):
        og.grad_close(ref + torch.tensor([0.0, 1e-9, 0.0], dtype=torch.float64), ref, scale, 1)   # small entry wrong
    with pytest.raises(AssertionError):
        og.grad_close(ref + torch.tensor([0.0, 0.0, 1e-30], dtype=torch.float64), ref, scale, 1)  # zero must be zero


def test_interp_bounds_cover_fp32_evaluation():
    """The bounds hold for an fp32 evaluation of the same graph (a CPU stand-in for the kernels' arithmetic)."""
    rng = np.random.default_rng(9)
    S = (6, 7, 5)
    vol = rng.standard_normal(S + (2,)).astype(F32)
    loc = _planted_loc(rng, S, (8, 9), 2.0)
    gout = rng.standard_normal((8, 9, 2)).astype(F32)
    for method, fill in (('linear', None), ('linear', 0.5), ('nearest', None)):
        res = []
        for dt in (torch.float32, torch.float64):
            v = torch.from_numpy(vol).to(dt).requires_grad_(True)
            l = torch.from_numpy(loc).to(dt).requires_grad_(True)
            og.torch_interpn(v, l, method, fill).backward(torch.from_numpy(gout).to(dt))
            res.append((v.grad, l.grad if l.grad is not None else torch.zeros_like(l)))
        vs, vk, ls, lk = og.interpn_grad_bounds(torch.from_numpy(vol), torch.from_numpy(loc), method, fill,
                                                torch.from_numpy(gout))
        og.grad_close(res[0][0], res[1][0], vs, vk, what='vol ' + method)
        og.grad_close(res[0][1], res[1][1], ls, lk, what='loc ' + method)
