"""
GPU gradient tests (SURVEY.md 8f item 1).  The reference gets its gradients from TensorFlow
autodiff of the op graph; here the same graph is written in differentiable torch float64
(floor: zero grad; clamp: passes on the closed interval, like tf.clip_by_value; gather:
scatter-add) and torch.autograd provides the expected gradients.

The cases further down compare every backward kernel path against the fp64 reference graphs
of oracle/grad.py, element by element within the bound of oracle.grad.grad_close.
"""

import numpy as np
import pytest
import torch

from oracle import grad as og

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ne(cuda):
    import neurite_b200
    return neurite_b200


@pytest.mark.parametrize('shape,C', [((6, 7, 8), 1), ((5, 6, 9), 3), ((9, 10), 2), ((17,), 1), ((10, 12, 36), 1),
                                     ((19, 9, 64), 1)])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', 0.5), ('nearest', None)])
def test_warp_and_interpn_gradients(ne, shape, C, method, fill):
    g = torch.Generator().manual_seed(len(shape) * 10 + C)
    D = len(shape)
    vol = torch.randn((2,) + shape + (C,), generator=g, dtype=torch.float64)
    # keep sample points away from integer coordinates (kinks) except a few exact edges
    flow = (torch.rand((2,) + shape + (D,), generator=g, dtype=torch.float64) * 5 - 2.5)
    grid = torch.stack(torch.meshgrid(*[torch.arange(s, dtype=torch.float64) for s in shape], indexing='ij'), -1)
    loc = grid[None] + flow
    frac = loc - torch.floor(loc)
    flow = flow + ((frac < 0.05).double() * 0.1 - (frac > 0.95).double() * 0.1)
    flow = flow.float().double()
    gout = torch.randn((2,) + shape + (C,), generator=g, dtype=torch.float64).float().double()
    vol = vol.float().double()

    v_ref = vol.clone().requires_grad_(True)
    f_ref = flow.clone().requires_grad_(True)
    out_ref = torch.stack([og.torch_interpn(v_ref[b], grid + f_ref[b], method, fill) for b in range(2)])
    out_ref.backward(gout)

    v = vol.float().cuda().requires_grad_(True)
    f = flow.float().cuda().requires_grad_(True)
    out = ne.layers.SpatialTransformer(interp_method=method, fill_value=fill)([v, f])
    np.testing.assert_allclose(out.detach().cpu().numpy(), out_ref.detach().numpy(), rtol=1e-5, atol=1e-5)
    out.backward(gout.float().cuda())
    np.testing.assert_allclose(v.grad.cpu().numpy(), v_ref.grad.numpy(), rtol=1e-4, atol=1e-4)
    f_exp = f_ref.grad.numpy() if f_ref.grad is not None else np.zeros(f_ref.shape)   # nearest: no gradient to loc
    np.testing.assert_allclose(f.grad.cpu().numpy(), f_exp, rtol=1e-4, atol=1e-4)

    # interpn with an explicit loc tensor
    v2 = vol[0].float().cuda().requires_grad_(True)
    l2 = (grid + flow[0]).float().cuda().requires_grad_(True)
    o2 = ne.utils.interpn(v2, l2, method, fill)
    o2.backward(gout[0].float().cuda())
    v3 = vol[0].clone().requires_grad_(True)
    l3 = (grid + flow[0]).float().double().requires_grad_(True)
    og.torch_interpn(v3, l3, method, fill).backward(gout[0])
    np.testing.assert_allclose(v2.grad.cpu().numpy(), v3.grad.numpy(), rtol=1e-4, atol=1e-4)
    l_exp = l3.grad.numpy() if l3.grad is not None else np.zeros(l3.shape)
    np.testing.assert_allclose(l2.grad.cpu().numpy(), l_exp, rtol=1e-4, atol=1e-4)


def test_resize_gradient(ne):
    g = torch.Generator().manual_seed(3)
    x = torch.randn((2, 5, 6, 7, 3), generator=g)
    xg = x.cuda().requires_grad_(True)
    out = ne.layers.Resize([2, 1.5, 0.8])(xg)
    gout = torch.randn(out.shape, generator=g)
    out.backward(gout.cuda())
    # expected: the same sampling expressed through interpn_torch on the linspace grid
    xr = x.double().requires_grad_(True)
    M = out.shape[1:-1]
    lin = []
    for d in range(3):
        S, m = x.shape[1 + d], M[d]
        delta = np.float32(S - 1) / np.float32(m - 1)
        v = (delta * np.arange(m, dtype=np.float32)).astype(np.float32)
        v[-1] = S - 1
        lin.append(torch.from_numpy(v).double())
    grid = torch.stack(torch.meshgrid(*lin, indexing='ij'), -1)
    ref = torch.stack([og.torch_interpn(xr[b], grid) for b in range(2)])
    ref.backward(gout.double())
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref.detach().numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(xg.grad.cpu().numpy(), xr.grad.numpy(), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('laplace', [0.0, 0.1])
def test_dice_gradient(ne, laplace):
    g = torch.Generator().manual_seed(5)
    L = 5
    lab = torch.randint(0, 4, (2, 6, 7, 8), generator=g)              # label 4 absent: 0/0 -> 0, zero gradient
    t = torch.nn.functional.one_hot(lab, L).double()
    p = torch.softmax(torch.randn((2, 6, 7, 8, L), generator=g, dtype=torch.float64), -1)
    p[..., 4] = 0
    w = torch.rand((1, L), generator=g, dtype=torch.float64)
    pr = p.clone().requires_grad_(True)
    top = 2 * (t * pr).flatten(1, 3).sum(1)
    bot = (t * t).flatten(1, 3).sum(1) + (pr * pr).flatten(1, 3).sum(1)
    dice = (top + laplace) / (bot + laplace) if laplace > 0 else torch.where(bot != 0, top / torch.where(bot != 0, bot, torch.ones_like(bot)), torch.zeros_like(top))
    (-(dice * w).mean()).backward()
    pg = p.float().cuda().requires_grad_(True)
    loss = ne.losses.Dice(weights=w.float().numpy(), laplace_smoothing=laplace).mean_loss(t.float().cuda(), pg)
    loss.backward()
    np.testing.assert_allclose(float(loss), float(-(dice * w).mean()), rtol=1e-5)
    np.testing.assert_allclose(pg.grad.cpu().numpy(), pr.grad.numpy(), rtol=1e-4, atol=1e-7)


@pytest.mark.parametrize('kw', [dict(), dict(from_logits=True), dict(label_smoothing=0.1), dict(reduction='sum'),
                                dict(reduction='none')])
def test_cce_gradient(ne, kw):
    g = torch.Generator().manual_seed(7)
    C = 6
    t = torch.nn.functional.one_hot(torch.randint(0, C, (2, 5, 6), generator=g), C).double()
    p = torch.rand((2, 5, 6, C), generator=g, dtype=torch.float64) + 0.05
    p[0, 0, 0] = torch.tensor([1.0, 0, 0, 0, 0, 0])                  # clipped entries: gradient masked
    lw = torch.rand(C, generator=g, dtype=torch.float64) + 0.5
    sw = torch.rand((2, 5, 6), generator=g, dtype=torch.float64) + 0.5
    pr = p.clone().requires_grad_(True)
    tt = t * lw
    ls = kw.get('label_smoothing', 0.0)
    if ls:
        tt = tt * (1 - ls) + ls / C
    if kw.get('from_logits'):
        l = -(tt * torch.log_softmax(pr, -1)).sum(-1)
    else:
        q = pr / pr.sum(-1, keepdim=True)
        l = -(tt * torch.log(torch.clamp(q, 1e-7, 1 - 1e-7))).sum(-1)
    l = l * sw
    red = kw.get('reduction', 'sum_over_batch_size')
    gper = torch.rand((2, 5, 6), generator=g, dtype=torch.float64)
    if red == 'none':
        l.backward(gper)
    else:
        (l.sum() if red == 'sum' else l.mean()).backward()
    pg = p.float().cuda().requires_grad_(True)
    c = ne.losses.CategoricalCrossentropy(label_weights=lw.float().numpy(), **kw)
    out = c(t.float().cuda(), pg, sample_weight=sw.float().cuda())
    if red == 'none':
        out.backward(gper.float().cuda())
    else:
        out.backward()
    np.testing.assert_allclose(pg.grad.cpu().numpy(), pr.grad.numpy(), rtol=2e-4, atol=1e-6)


def test_lc3d_gradient(ne):
    """LocallyConnected3D gradients vs torch autograd of an unfold + einsum formulation."""
    g = torch.Generator().manual_seed(9)
    B, I, Cin, Cout = 3, (6, 7, 8), 4, 8
    x = torch.randn((B,) + I + (Cin,), generator=g)
    lay = ne.layers.LocallyConnected3D(Cout, 3, activation='tanh')
    lay.build(x.shape)
    O = (lay.output_row, lay.output_col, lay.output_z)
    with torch.no_grad():
        lay.kernel.normal_(0, 0.2, generator=g)
        lay.bias.normal_(0, 1, generator=g)
    k_ref = lay.kernel.detach().double().clone().requires_grad_(True)
    b_ref = lay.bias.detach().double().clone().requires_grad_(True)
    x_ref = x.double().clone().requires_grad_(True)
    win = x_ref.unfold(1, 3, 1).unfold(2, 3, 1).unfold(3, 3, 1)            # [B,o0,o1,o2,Cin,k0,k1,k2]
    patches = win.permute(0, 1, 2, 3, 5, 6, 7, 4).reshape(B, -1, 27 * Cin)  # j = ((i0*3+i1)*3+i2)*Cin + c
    ref = torch.tanh(torch.einsum('bpj,pjf->bpf', patches, k_ref).reshape((B,) + O + (Cout,)) + b_ref)
    gout = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    ref.backward(gout)
    lay.cuda()
    xg = x.cuda().requires_grad_(True)
    out = lay(xg)
    np.testing.assert_allclose(out.detach().cpu().numpy(), ref.detach().numpy(), rtol=1e-4, atol=1e-5)
    out.backward(gout.float().cuda())
    np.testing.assert_allclose(xg.grad.cpu().numpy(), x_ref.grad.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(lay.kernel.grad.cpu().numpy(), k_ref.grad.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(lay.bias.grad.cpu().numpy(), b_ref.grad.numpy(), rtol=1e-4, atol=1e-4)


# =======================================================================================
# every backward path against the fp64 reference graphs (oracle/grad.py), element by element
# =======================================================================================
def _g(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _plant(flow, frac=0.06, seed=0):
    """Overwrite flow [B, *S, D] so that, on a random subset of voxels and axes, the fp32 location coord + flow
    is an exact integer, an exact half, exactly 0, exactly S-1, or just outside the volume."""
    S = flow.shape[1:-1]
    D = len(S)
    g = _g(seed)
    grid = og.warp_loc(torch.zeros_like(flow[0]))
    for d in range(D):
        n = S[d]
        pick = torch.rand(flow.shape[:-1], generator=g, device=flow.device) < frac
        kind = torch.randint(0, 6, flow.shape[:-1], generator=g, device=flow.device)
        integer = torch.randint(0, n, flow.shape[:-1], generator=g, device=flow.device).float()
        target = torch.stack([integer, integer + 0.5 if n > 1 else integer, torch.zeros_like(integer),
                              torch.full_like(integer, n - 1), torch.full_like(integer, -0.25),
                              torch.full_like(integer, n - 0.75)])
        target = torch.gather(target, 0, kind[None])[0]
        flow[..., d] = torch.where(pick, target - grid[..., d], flow[..., d])
    return flow


def _warp_ref(vol, flow, gout, method, fill):
    v = vol.double().requires_grad_(True)
    f = flow.double().requires_grad_(True)
    og.torch_warp(v, f, method, fill).backward(gout.double())
    gf = f.grad if f.grad is not None else torch.zeros_like(f)
    return v.grad, gf, og.warp_grad_bounds(vol, flow, method, fill, gout)


def _warp_check(ne, vol, flow, gout, method, fill, ref, requests=('both', 'vol', 'flow'), tag=''):
    gv_ref, gf_ref, (vs, vk, fs, fk) = ref
    for req in requests:
        v = vol.clone().requires_grad_(req != 'flow')
        f = flow.clone().requires_grad_(req != 'vol')
        ne.layers.SpatialTransformer(interp_method=method, fill_value=fill)([v, f]).backward(gout)
        if req != 'flow':
            og.grad_close(v.grad, gv_ref, vs, vk, what='%s %s d/dvol' % (tag, req))
        else:
            assert v.grad is None
        if req != 'vol':
            og.grad_close(f.grad, gf_ref, fs, fk, what='%s %s d/dflow' % (tag, req))
        else:
            assert f.grad is None


FLOWS = {'iid2.5': (2.5, None), 'iid7': (7.0, None), 'shift': (1.0, (9.3, -7.6, 11.2))}


@pytest.mark.parametrize('family', list(FLOWS))
@pytest.mark.parametrize('shape', [(20, 17, 100), (9, 24, 36)])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', -1.5), ('nearest', None), ('nearest', -1.5)])
def test_warp_c1_tiled_backward_vs_fp64_reference(ne, monkeypatch, shape, family, method, fill):
    """D=3, C=1, W % 4 == 0: warp3d_bwd_tile_kernel (corners outside the staged box through bwd_global3) and, with
    NRT_WARP_BWD_TILE=0, warp_bwd_kernel -- both against the reference, for vol+flow, vol-only and flow-only."""
    amp, shift = FLOWS[family]
    g = _g(100 * list(FLOWS).index(family) + shape[0])             # deterministic across processes
    vol = torch.randn((3,) + shape + (1,), generator=g, device='cuda')
    flow = (torch.rand((3,) + shape + (3,), generator=g, device='cuda') * 2 - 1) * amp
    if shift is not None:
        flow = flow + torch.tensor(shift, device='cuda')
    flow = _plant(flow, seed=len(family))
    gout = torch.randn((3,) + shape + (1,), generator=g, device='cuda')
    ref = _warp_ref(vol, flow, gout, method, fill)
    for tile in ('1', '0'):
        monkeypatch.setenv('NRT_WARP_BWD_TILE', tile)
        _warp_check(ne, vol, flow, gout, method, fill, ref, tag='tile=' + tile)


@pytest.mark.parametrize('shape,C', [((7, 9, 30), 1), ((7, 9, 30), 2), ((6, 5, 30), 3), ((5, 6, 30), 16),
                                     ((11, 30), 2), ((13, 30), 16), ((30,), 3), ((30,), 1)])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', -1.5), ('nearest', None), ('nearest', -1.5)])
def test_warp_generic_backward_vs_fp64_reference(ne, shape, C, method, fill):
    """warp_bwd_kernel: W = 30 (not a multiple of 4), C in {1, 2, 3, 16}, D = 3, 2, 1, planted edge locations."""
    g = _g(len(shape) * 100 + C)
    D = len(shape)
    vol = torch.randn((2,) + shape + (C,), generator=g, device='cuda')
    flow = _plant((torch.rand((2,) + shape + (D,), generator=g, device='cuda') * 2 - 1) * 4, frac=0.1, seed=C)
    gout = torch.randn((2,) + shape + (C,), generator=g, device='cuda')
    _warp_check(ne, vol, flow, gout, method, fill, _warp_ref(vol, flow, gout, method, fill))


def test_warp_full_size_cfg2_backward_vs_fp64_reference(ne):
    """cfg 2: 160x192x224, C=1, linear, i.i.d. +-3 (the reference graph runs on the GPU in fp64)."""
    g = _g(2)
    shape = (160, 192, 224)
    vol = torch.randn((1,) + shape + (1,), generator=g, device='cuda')
    flow = (torch.rand((1,) + shape + (3,), generator=g, device='cuda') * 2 - 1) * 3
    gout = torch.randn((1,) + shape + (1,), generator=g, device='cuda')
    _warp_check(ne, vol, flow, gout, 'linear', None, _warp_ref(vol, flow, gout, 'linear', None), requests=('both',))


def test_vec_int_backward_vs_fp64_reference(ne):
    """VecInt(int_steps=5): five chained C=3 warp backward launches with the same tensor as vol and flow."""
    g = _g(5)
    vel = (torch.rand((2, 10, 12, 14, 3), generator=g, device='cuda') * 2 - 1) * 12
    gout = torch.randn(vel.shape, generator=g, device='cuda')
    v = vel.clone().requires_grad_(True)
    ne.layers.VecInt(int_steps=5)(v).backward(gout)
    vr = vel.double().requires_grad_(True)
    og.torch_vec_int(vr, 5).backward(gout.double())
    scale, k = og.vec_int_grad_bounds(vel, 5, gout)
    og.grad_close(v.grad, vr.grad, scale, k, what='VecInt d/dvel')


@pytest.mark.parametrize('S', [(23,), (9, 11), (6, 7, 9)])
@pytest.mark.parametrize('C', [1, 4, 5])
@pytest.mark.parametrize('method,fill', [('linear', None), ('linear', 0.5), ('nearest', None), ('nearest', 0.5)])
def test_interpn_backward_vs_fp64_reference(ne, S, C, method, fill):
    """interpn_bwd_kernel on scattered [N, D] locations inside and outside the volume (exact integers, halves,
    0 and S-1 planted) and on a grid-shaped [*S, D] location tensor."""
    g = _g(len(S) * 10 + C)
    D = len(S)
    vol = torch.randn(S + (C,), generator=g, device='cuda')
    hi = torch.tensor(S, device='cuda', dtype=torch.float32) - 1
    scattered = torch.rand((301, D), generator=g, device='cuda') * (hi + 4) - 2
    special = torch.tensor([0.0, 1.0, 0.5, -0.25], device='cuda')
    edge = torch.stack([torch.cat([special, hi[d:d + 1], hi[d:d + 1] - 0.5, hi[d:d + 1] + 0.25]) for d in range(D)], -1)
    scattered = torch.cat([scattered, edge, torch.floor(scattered[:40]) + 0.5, torch.round(scattered[40:80])])
    grid = _plant((torch.rand((1,) + S + (D,), generator=g, device='cuda') * 2 - 1) * 3, frac=0.1, seed=D)[0] \
        + og.warp_loc(torch.zeros(S + (D,), device='cuda'))
    for loc in (scattered, grid):
        gout = torch.randn(loc.shape[:-1] + (C,), generator=g, device='cuda')
        v = vol.clone().requires_grad_(True)
        l = loc.clone().requires_grad_(True)
        ne.utils.interpn(v, l, method, fill).backward(gout)
        vr = vol.double().requires_grad_(True)
        lr = loc.double().requires_grad_(True)
        og.torch_interpn(vr, lr, method, fill).backward(gout.double())
        vs, vk, ls, lk = og.interpn_grad_bounds(vol, loc, method, fill, gout)
        og.grad_close(v.grad, vr.grad, vs, vk, what='interpn d/dvol')
        og.grad_close(l.grad, lr.grad if lr.grad is not None else torch.zeros_like(lr), ls, lk, what='interpn d/dloc')


def test_interpn_4d_gradient_raises(ne):
    vol = torch.randn((3, 4, 5, 6, 1), device='cuda', requires_grad=True)
    loc = torch.rand((10, 4), device='cuda') * 2
    with torch.no_grad():
        assert ne.utils.interpn(vol, loc).shape == (10, 1)            # the 4-D forward is built
    with pytest.raises(NotImplementedError, match='interpn gradients are built for up to'):
        ne.utils.interpn(vol, loc)


RESIZE_CASES = [((9,), 1, 2), ((10,), 3, 0.5), ((3,), 4, 1.7),
                ((6, 7), 3, [2, 0.5]), ((3, 5), 1, [1.7, 0.4]), ((7, 3), 4, [0.5, 0.5]),
                ((4, 5, 3), 3, [1.5, 2, 3.7]), ((3, 6, 5), 1, [1.7, 0.5, 0.4]), ((5, 3, 4), 4, [2, 0.34, 0.5]),
                ((40, 48, 56), 3, 2)]


@pytest.mark.parametrize('shape,C,zoom', RESIZE_CASES)
@pytest.mark.parametrize('method', ['linear', 'nearest'])
def test_resize_backward_vs_fp64_reference(ne, shape, C, zoom, method):
    """resize_bwd_kernel: D = 1, 2, 3, up- and down-sampling, axes that become M = 1 and M = 2, exact half-integer
    nearest samples (1.7 on a size-3 axis: 5 samples at spacing 0.5), and a mid-size case for accumulation depth."""
    g = _g(len(shape) * 7 + C)
    x = torch.randn((2,) + shape + (C,), generator=g, device='cuda')
    xg = x.clone().requires_grad_(True)
    out = ne.layers.Resize(zoom, interp_method=method)(xg)
    gout = torch.randn(out.shape, generator=g, device='cuda')
    out.backward(gout)
    xr = x.double().requires_grad_(True)
    ref = og.torch_resize(xr, zoom, method)
    assert ref.shape == out.shape
    ref.backward(gout.double())
    scale, k = og.resize_grad_bounds(x, zoom, method, gout)
    og.grad_close(xg.grad, xr.grad, scale, k, what='resize d/dx')


def _dice_ref(t, p, laplace, entry, w, gup):
    tr, pr = t.double().requires_grad_(True), p.double().requires_grad_(True)
    d = og.torch_dice(tr, pr, laplace)
    d.retain_grad()
    if entry == 'dice':
        d.backward(gup.double())
    else:
        m = (d * w.double()).mean()
        (m if entry == 'mean_dice' else -m).backward()
    return tr.grad, pr.grad, d.grad


def _dice_check(ne, t, p, laplace, entry, w, gup, tag=''):
    tg, pg = t.detach().requires_grad_(True), p.detach().requires_grad_(True)      # keeps a view's offset
    m = ne.losses.Dice(weights=w.cpu().numpy(), laplace_smoothing=laplace)
    out = m.dice(tg, pg) if entry == 'dice' else getattr(m, entry)(tg, pg)
    out.backward(gup if entry == 'dice' else None)
    gt_ref, gp_ref, G = _dice_ref(t, p, laplace, entry, w, gup)
    sp, st, k = og.dice_grad_bounds(t, p, G, laplace)
    og.grad_close(pg.grad, gp_ref, sp, k, what='%s dice d/dy_pred' % tag)
    og.grad_close(tg.grad, gt_ref, st, k, what='%s dice d/dy_true' % tag)


def _dice_inputs(g, B, S, L, absent=True):
    lab = torch.randint(0, max(L - 1, 1) if absent else L, (B,) + S, generator=g, device='cuda')
    t = torch.nn.functional.one_hot(lab, L).float()
    p = torch.softmax(torch.randn((B,) + S + (L,), generator=g, device='cuda'), -1)
    if absent and L > 1:
        p[..., L - 1] = 0                                    # absent label: bot == 0 without laplace
    return t, p


@pytest.mark.parametrize('L', [1, 3, 4, 5, 16, 20, 64])
@pytest.mark.parametrize('laplace', [0.0, 0.1])
def test_dice_backward_vs_fp64_reference(ne, L, laplace):
    """dice_bwd_kernel: float4 branch (L % 4 == 0) and scalar branch, absent labels, batch 1 and 3, random upstream
    gradients through dice / mean_dice / mean_loss with weights, gradients w.r.t. y_pred and y_true."""
    g = _g(L * 3 + int(laplace * 10))
    for B, entry in ((3, 'dice'), (1, 'mean_dice'), (3, 'mean_loss')):
        t, p = _dice_inputs(g, B, (5, 6, 7), L)
        w = torch.rand((1, L), generator=g, device='cuda')
        gup = torch.randn((B, L), generator=g, device='cuda')
        _dice_check(ne, t, p, laplace, entry, w, gup, tag='L=%d B=%d %s' % (L, B, entry))


def test_dice_backward_offset_view_and_grid_stride_wrap(ne):
    """L = 16 through a 4-byte-offset view (scalar branch), and 2x48x48x48x16 (the grid-stride loop wraps)."""
    g = _g(16)
    t, p = _dice_inputs(g, 2, (6, 7, 8), 16)
    bt = torch.empty(t.numel() + 1, device='cuda')
    bp = torch.empty(p.numel() + 1, device='cuda')
    tv, pv = bt[1:].view(t.shape), bp[1:].view(p.shape)
    tv.copy_(t)
    pv.copy_(p)
    assert tv.data_ptr() % 16 == 4 and tv.is_contiguous()
    w = torch.rand((1, 16), generator=g, device='cuda')
    gup = torch.randn((2, 16), generator=g, device='cuda')
    _dice_check(ne, tv, pv, 0.0, 'dice', w, gup, tag='offset view')
    t, p = _dice_inputs(g, 2, (48, 48, 48), 16, absent=False)
    _dice_check(ne, t, p, 0.1, 'dice', w, gup, tag='2x48^3x16')


CCE_VARIANTS = {'plain': dict(), 'label_weights': dict(), 'sample_weights': dict(),
                'smoothing': dict(label_smoothing=0.1), 'from_logits': dict(from_logits=True)}


def _cce_inputs(g, rows, C, logits):
    t = torch.nn.functional.one_hot(torch.randint(0, C, rows, generator=g, device='cuda'), C).float()
    if logits:
        return t, torch.randn(rows + (C,), generator=g, device='cuda') * 2
    p = torch.rand(rows + (C,), generator=g, device='cuda') + 0.05
    flat = p.reshape(-1, C)
    flat[0] = 0
    flat[0, 0] = 1                                           # one-hot p: every entry clipped
    flat[3, 1] = 0                                           # p = 0: that entry clipped
    flat[5, :C // 2] = 0
    t.reshape(-1, C)[5] = 0
    t.reshape(-1, C)[5, 0] = 1                               # the true label of row 5 is clipped
    return t, p


def _cce_check(ne, t, p, lw, sw, kw, red, g, tag=''):
    n = p.numel() // p.shape[-1]
    pg = p.detach().requires_grad_(True)                                         # keeps a view's offset
    out = ne.losses.CategoricalCrossentropy(label_weights=lw, reduction=red, **kw)(t, pg, sample_weight=sw)
    up = torch.randn(out.shape, generator=g, device='cuda')
    out.backward(up)
    pr = p.double().requires_grad_(True)
    og.torch_cce(t.double(), pr, None if lw is None else lw.double(), None if sw is None else sw.double(),
                 reduction=red, **kw).backward(up.double())
    row = up.double() * (1.0 / n if red == 'sum_over_batch_size' else 1.0) * torch.ones(p.shape[:-1], device='cuda')
    if sw is not None:
        row = row * sw.double()
    scale, k = og.cce_grad_bounds(t, p, lw, row, kw.get('from_logits', False), kw.get('label_smoothing', 0.))
    og.grad_close(pg.grad, pr.grad, scale, k, what='%s cce d/dy_pred' % tag)


@pytest.mark.parametrize('C', [2, 3, 4, 5, 8, 12, 16, 32, 64, 128])
@pytest.mark.parametrize('variant', list(CCE_VARIANTS))
def test_cce_backward_vs_fp64_reference(ne, C, variant):
    """cce_bwd_vec4_kernel (C in {4..128} power of two, normalised) and cce_bwd_kernel, every reduction,
    154 rows (not a multiple of 256 / q), rows with clipped entries (p = 0 and one-hot p)."""
    g = _g(C * 11 + len(variant))
    kw = CCE_VARIANTS[variant]
    rows = (2, 7, 11)
    t, p = _cce_inputs(g, rows, C, kw.get('from_logits', False))
    lw = torch.rand(C, generator=g, device='cuda') + 0.5 if variant == 'label_weights' else None
    sw = torch.rand(rows, generator=g, device='cuda') + 0.5 if variant == 'sample_weights' else None
    for red in ('sum_over_batch_size', 'sum', 'none'):
        _cce_check(ne, t, p, lw, sw, kw, red, g, tag='C=%d %s %s' % (C, variant, red))


def test_cce_backward_scalar_kernel_for_misaligned_operands(ne):
    """C = 16 through a 4-byte-offset y_pred view, and with 4-byte-offset label weights: the scalar kernel."""
    g = _g(161)
    rows = (3, 50)
    t, p = _cce_inputs(g, rows, 16, False)
    buf = torch.empty(p.numel() + 1, device='cuda')
    pv = buf[1:].view(p.shape)
    pv.copy_(p)
    _cce_check(ne, t, pv, None, None, {}, 'sum', g, tag='offset y_pred')
    lbuf = torch.empty(17, device='cuda')
    lw = lbuf[1:]
    lw.copy_(torch.rand(16, generator=g, device='cuda') + 0.5)
    assert lw.data_ptr() % 16 == 4
    _cce_check(ne, t, p, lw, None, {}, 'none', g, tag='offset label weights')


LC3D_CASES = [(1, 3, 4, (3, 3, 3), (1, 1, 1), 'channels_last'),
              (2, 16, 16, (2, 3, 2), (2, 1, 2), 'channels_last'),
              (3, 3, 32, (3, 3, 3), (1, 1, 1), 'channels_first'),
              (4, 3, 128, (2, 3, 2), (2, 1, 2), 'channels_last'),
              (5, 16, 4, (3, 3, 3), (1, 1, 1), 'channels_first'),
              (8, 3, 16, (2, 3, 2), (2, 1, 2), 'channels_last'),
              (9, 3, 8, (3, 3, 3), (1, 1, 1), 'channels_last')]


def _lc3d_setup(g, B, Cin, Cout, ks, st, fmt, I=(6, 7, 8)):
    shape = (B, Cin) + I if fmt == 'channels_first' else (B,) + I + (Cin,)
    x = torch.randn(shape, generator=g, device='cuda')
    O = [(I[d] - ks[d]) // st[d] + 1 for d in range(3)]
    P, F = int(np.prod(O)), int(np.prod(ks)) * Cin
    k = torch.randn((P, F, Cout), generator=g, device='cuda') * 0.2
    b = torch.randn(tuple(O) + (Cout,), generator=g, device='cuda')
    return x, k, b, O


@pytest.mark.parametrize('B,Cin,Cout,ks,st,fmt', LC3D_CASES)
def test_lc3d_backward_vs_fp64_reference(ne, B, Cin, Cout, ks, st, fmt):
    """lc3d_bwd_kernel<4>/<2>/<1> pass sequences for B in {1,2,3,4,5,8,9} (grad_kernel accumulated over passes),
    Cout in {4,16,32,128}, strides, channels_first with its raw-reshape bias; x-and-kernel, x-only, kernel-only."""
    g = _g(B * 100 + Cout)
    x, k, b, O = _lc3d_setup(g, B, Cin, Cout, ks, st, fmt)
    ref_out = og.torch_local_conv3d(x.double(), k.double(), b.double(), ks, st, fmt)
    gout = torch.randn(ref_out.shape, generator=g, device='cuda')
    xr, kr, br = (t.double().requires_grad_(True) for t in (x, k, b))
    og.torch_local_conv3d(xr, kr, br, ks, st, fmt).backward(gout.double())
    xs, xk, kscale, kk = og.lc3d_grad_bounds(x, k, gout, ks, st, fmt)
    b0 = torch.zeros_like(br).requires_grad_(True)            # d out / d bias is 0/1: scale = sum_b |dy|
    bscale, = torch.autograd.grad(og.torch_local_conv3d(xr.detach(), kr.detach(), b0, ks, st, fmt), b0,
                                  gout.double().abs())
    for req in ('both', 'x', 'kernel'):
        lay = ne.layers.LocallyConnected3D(Cout, ks, strides=st, data_format=fmt)
        lay.build(x.shape)
        with torch.no_grad():
            lay.kernel.copy_(k.cpu())
            lay.bias.copy_(b.cpu())
        lay.cuda()
        lay.kernel.requires_grad_(req != 'x')
        lay.bias.requires_grad_(req != 'x')
        xg = x.clone().requires_grad_(req != 'kernel')
        lay(xg).backward(gout)
        if req != 'kernel':
            og.grad_close(xg.grad, xr.grad, xs, xk, what='lc3d %s d/dx' % req)
        if req != 'x':
            og.grad_close(lay.kernel.grad, kr.grad, kscale, kk, what='lc3d %s d/dkernel' % req)
            og.grad_close(lay.bias.grad, br.grad, bscale, B + 2, what='lc3d %s d/dbias' % req)


def test_lc3d_position_shards_and_implementations(ne):
    """Two p0 / p_count halves give the whole gradient; implementation 2 / 3 kernel gradients are the
    implementation-1 gradient in their layouts; Cout = 12 backward raises instead of returning something."""
    g = _g(77)
    B, Cin, Cout, ks, st, fmt = 5, 3, 8, (2, 3, 2), (2, 1, 2), 'channels_last'
    x, k, b, O = _lc3d_setup(g, B, Cin, Cout, ks, st, fmt)
    P = int(np.prod(O))
    gout = torch.randn((B, P, Cout), generator=g, device='cuda')
    xs, xk, kscale, kk = og.lc3d_grad_bounds(x, k, gout.reshape((B,) + tuple(O) + (Cout,)), ks, st, fmt)
    half = P // 2 + 1
    gx_sum = torch.zeros_like(x)
    gk_parts = []
    for p0, pc in ((0, half), (half, P - half)):
        xg = x.clone().requires_grad_(True)
        kg = k[p0:p0 + pc].clone().requires_grad_(True)
        ne.layers.local_conv3d(xg, kg, None, ks, st, O, fmt, None, p0, pc).backward(gout[:, p0:p0 + pc].contiguous())
        xr, kr = x.double().requires_grad_(True), k[p0:p0 + pc].double().requires_grad_(True)
        og.torch_local_conv3d(xr, kr, None, ks, st, fmt, p0, pc).backward(gout[:, p0:p0 + pc].double())
        og.grad_close(kg.grad, kr.grad, kscale[p0:p0 + pc], kk[p0:p0 + pc], what='shard d/dkernel')
        gx_sum += xg.grad
        gk_parts.append(kg.grad)
    xr, kr = x.double().requires_grad_(True), k.double().requires_grad_(True)
    og.torch_local_conv3d(xr, kr, None, ks, st, fmt).backward(gout.reshape((B,) + tuple(O) + (Cout,)).double())
    og.grad_close(gx_sum, xr.grad, xs, xk + 1, what='shards d/dx')
    og.grad_close(torch.cat(gk_parts), kr.grad, kscale, kk, what='shards d/dkernel')

    grads = {}
    for impl in (1, 2, 3):
        lay = ne.layers.LocallyConnected3D(Cout, ks, strides=st, implementation=impl)
        lay.build(x.shape)
        with torch.no_grad():
            lay.kernel.copy_(ne.layers.lc3d_kernel_to_impl(k.cpu(), impl, x.shape[1:4], Cin, ks, st))
        lay.cuda()
        lay(x).backward(gout.reshape((B,) + tuple(O) + (Cout,)))
        grads[impl] = lay.kernel.grad
    og.grad_close(grads[1], kr.grad, kscale, kk, what='impl 1 d/dkernel')
    for impl in (2, 3):
        assert torch.equal(grads[impl], ne.layers.lc3d_kernel_to_impl(grads[1], impl, x.shape[1:4], Cin, ks, st))

    lay = ne.layers.LocallyConnected3D(12, ks, strides=st)
    lay.build(x.shape)
    lay.cuda()
    out = lay(x.clone().requires_grad_(True))
    with pytest.raises(Exception, match='lc3d backward is built for Cout'):
        out.sum().backward()


def test_backward_dispatch_reaches_each_kernel(ne, monkeypatch):
    """The path tests above rely on the dispatch: record which kernels representative cases launch."""
    from torch.profiler import profile, ProfilerActivity

    def names(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    g = _g(3)
    probe = names(lambda: torch.ones(4, device='cuda').add_(1))
    if not probe:
        pytest.skip('torch.profiler recorded no CUDA events on this machine')

    def warp(shape, C):
        v = torch.randn((1,) + shape + (C,), device='cuda', requires_grad=True)
        f = (torch.rand((1,) + shape + (len(shape),), generator=g, device='cuda') * 4 - 2).requires_grad_(True)
        return lambda: ne.layers.SpatialTransformer()([v, f]).sum().backward()

    def has(ns, s):
        return any(s in n for n in ns)

    ns = names(warp((9, 24, 36), 1))
    assert has(ns, 'warp3d_bwd_tile_kernel') and not has(ns, 'warp_bwd_kernel'), ns
    monkeypatch.setenv('NRT_WARP_BWD_TILE', '0')
    ns = names(warp((9, 24, 36), 1))
    assert has(ns, 'warp_bwd_kernel') and not has(ns, 'warp3d_bwd_tile_kernel'), ns
    monkeypatch.delenv('NRT_WARP_BWD_TILE')
    ns = names(warp((7, 9, 30), 1))
    assert has(ns, 'warp_bwd_kernel') and not has(ns, 'warp3d_bwd_tile_kernel'), ns

    def cce(C, logits):
        t, p = _cce_inputs(g, (3, 5), C, logits)
        p.requires_grad_(True)
        return lambda: ne.losses.CategoricalCrossentropy(from_logits=logits)(t, p).backward()

    ns = names(cce(16, False))
    assert has(ns, 'cce_bwd_vec4_kernel') and not has(ns, 'cce_bwd_kernel('), ns
    for C, logits in ((12, False), (16, True)):
        ns = names(cce(C, logits))
        assert has(ns, 'cce_bwd_kernel') and not has(ns, 'cce_bwd_vec4_kernel'), ns

    for B, want in ((9, ['lc3d_bwd_kernel<4>', 'lc3d_bwd_kernel<1>']), (3, ['lc3d_bwd_kernel<2>', 'lc3d_bwd_kernel<1>']),
                    (2, ['lc3d_bwd_kernel<2>'])):
        x, k, b, O = _lc3d_setup(g, B, 3, 8, (3, 3, 3), (1, 1, 1), 'channels_last')
        kg = k.clone().requires_grad_(True)
        ns = names(lambda: ne.layers.local_conv3d(x, kg, None, (3, 3, 3), (1, 1, 1), O).sum().backward())
        got = sorted({s for s in ('lc3d_bwd_kernel<4>', 'lc3d_bwd_kernel<2>', 'lc3d_bwd_kernel<1>') if has(ns, s)})
        assert got == sorted(want), (B, ns)
        if B == 9:
            assert sum('lc3d_bwd_kernel<4>' in n for n in ns) == 2, ns

    x = torch.randn((2, 5, 6, 7, 3), device='cuda', requires_grad=True)
    ns = names(lambda: ne.layers.Resize(2, interp_method='nearest')(x).sum().backward())
    assert has(ns, 'resize_bwd_kernel'), ns
    v = torch.randn((6, 7, 9, 4), device='cuda', requires_grad=True)
    loc = (torch.rand((50, 3), generator=g, device='cuda') * 6).requires_grad_(True)
    ns = names(lambda: ne.utils.interpn(v, loc).sum().backward())
    assert has(ns, 'interpn_bwd_kernel'), ns
