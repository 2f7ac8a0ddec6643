"""
Differentiable torch restatements of the reference graphs: the GRADIENT oracle.  TEST
INFRASTRUCTURE (see oracle/__init__.py).

TensorFlow gets the reference's gradients by autodiff of the op graph; each function here
writes the same graph in torch, op for op, so torch.autograd differentiates it the same way
(floor / round: zero gradient; clip_by_value and torch.clamp: the gradient passes on the
CLOSED interval; gather: scatter-add; divide_no_nan: zero where the denominator is zero).
They work in whatever dtype they are given:

  * float32: the interpolation graphs (interpn, warp, resize, vec_int) reproduce the numpy
    oracle (oracle/interp.py) bit for bit -- tests/test_oracle_grad.py checks it;
  * float64: the gradient reference.  Sample locations are formed in fp32 first (coord +
    flow, tf.linspace), exactly as the kernels and TF do, and only then promoted, and the
    per-axis interpolation weights keep the value the fp32 graph gives them (f1 - x and
    1 - w are each one fp32 rounding there); products and sums are then fp64.

Next to the graphs are the per-element error bounds the gradient tests use (grad_close):

    |got - ref| <= c * k * 2^-24 * scale      element by element

scale is the sum of the absolute values of the terms that make up that gradient element and
k the number of fp32 operations accumulated into it.  The kernels' fp32 atomics make the
summation order nondeterministic, so this is the bound any order satisfies (c <= 4).
"""
import itertools

import numpy as np
import torch

from .interp import tf_linspace_f32

U = 2.0 ** -24


def grad_close(got, ref, scale, k, c=4.0, what='gradient', approx=0.):
    """Assert |got - ref| <= c * k * 2^-24 * scale + approx element by element (k, approx: scalar or per element).
    approx is the documented error of an approximate hardware function (oracle/forward.py names each one); it is
    0 for every gradient."""
    got = got.detach().to(torch.float64)
    ref = ref.detach().to(device=got.device, dtype=torch.float64)
    scale = torch.as_tensor(scale, dtype=torch.float64, device=got.device)
    k = torch.as_tensor(k, dtype=torch.float64, device=got.device)
    approx = torch.as_tensor(approx, dtype=torch.float64, device=got.device)
    assert c <= 4
    assert bool((approx >= 0).all())
    assert got.shape == ref.shape, '%s: shape %s vs reference %s' % (what, tuple(got.shape), tuple(ref.shape))
    tol = c * k * U * scale + approx
    err = (got - ref).abs()
    bad = ~(err <= tol)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        ratio = (err / tol.clamp_min(1e-300)).reshape(-1)
        j = int(torch.argmax(torch.where(torch.isfinite(ratio), ratio, torch.full_like(ratio, np.inf))))
        idx = lambda n: tuple(int(v) for v in np.unravel_index(n, tuple(got.shape)))   # noqa: E731
        tb = lambda t, n: float(torch.broadcast_to(t, got.shape).reshape(-1)[n])         # noqa: E731
        raise AssertionError(
            '%s: %d of %d elements outside c*k*2^-24*scale + approx; first at %s: got %.9g ref %.9g tol %.3g '
            '(scale %.3g k %g); '
            'worst at %s: got %.9g ref %.9g tol %.3g'
            % (what, int(bad.sum()), bad.numel(), idx(i), float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]),
               tb(tol, i), tb(scale, i), tb(k, i), idx(j), float(got.reshape(-1)[j]), float(ref.reshape(-1)[j]),
               tb(tol, j)))


def _f32_valued(t):
    """t carrying the value of one fp32 rounding of t, with t's derivative (identity in fp32)."""
    if t.dtype == torch.float32:
        return t
    return t + (t.float().to(t.dtype) - t).detach()


def _strides(S):
    return [int(np.prod(S[d + 1:])) for d in range(len(S))]


def _linear_axes(loc, S, f32_steps=True):
    """Per-axis corners and weights of the linear interpolation (utils.py:139-155):
    x = clip(loc), f0 = clip(floor(loc)), f1 = clip(f0 + 1), w(bit 0) = f1 - x, w(bit 1) = 1 - w(bit 0).
    f32_steps=False keeps the weights in the working dtype (same derivative; for finite-difference checks)."""
    rnd = _f32_valued if f32_steps else (lambda t: t)
    axes = []
    for d in range(loc.shape[-1]):
        mx = float(S[d] - 1)
        x = torch.clamp(loc[..., d], 0, mx)
        f0 = torch.clamp(torch.floor(loc[..., d]), 0, mx)
        f1 = torch.clamp(f0 + 1, 0, mx)
        wlo = rnd(f1 - x)
        whi = rnd(1 - wlo)
        axes.append(((f0.long(), f1.long()), (wlo, whi)))
    return axes


def _corners(axes, strides):
    """(flat index, prod_n weight, per-axis bits) of each cube corner, in the reference's order."""
    D = len(axes)
    for bits in itertools.product([0, 1], repeat=D):
        idx = sum(axes[d][0][bits[d]] * strides[d] for d in range(D))
        w = axes[0][1][bits[0]]
        for d in range(1, D):
            w = w * axes[d][1][bits[d]]
        yield idx, w, bits


def _oob(loc, S):
    oob = torch.zeros_like(loc[..., 0], dtype=torch.bool)
    for d in range(loc.shape[-1]):
        oob = oob | (loc[..., d] < 0) | (loc[..., d] > S[d] - 1)
    return oob


def torch_interpn(vol, loc, method='linear', fill=None, f32_steps=True):
    """utils.py:73-220 (interpn) for vol [*S, C] and loc [*O, D] of vol's dtype -> [*O, C]."""
    S = vol.shape[:-1]
    flat = vol.reshape(-1, vol.shape[-1])
    strides = _strides(S)
    if method == 'linear':
        out = 0
        for idx, w, _ in _corners(_linear_axes(loc, S, f32_steps), strides):
            out = out + w[..., None] * flat[idx]
    else:
        assert method == 'nearest', method
        r = [torch.clamp(torch.round(loc[..., d]).long(), 0, S[d] - 1) for d in range(loc.shape[-1])]
        out = flat[sum(r[d] * strides[d] for d in range(len(r)))]
    if fill is not None:
        oob = _oob(loc, S)[..., None]
        out = out * (~oob).to(out.dtype) + oob.to(out.dtype) * fill
    return out


def warp_loc(flow, f32_steps=True):
    """Sample locations of a dense warp, flow [*S, D], in flow's dtype.  The value is the fp32 sum ndgrid + flow
    (what the kernels and TF compute); the derivative w.r.t. flow is the identity in flow's dtype, so an fp64
    gradient is not rounded to fp32 on its way back to flow.  f32_steps=False: the plain sum in flow's dtype,
    for finite-difference checks."""
    S = flow.shape[:-1]
    grid = torch.stack(torch.meshgrid(*[torch.arange(s, dtype=flow.dtype, device=flow.device) for s in S],
                                      indexing='ij'), -1)
    loc = grid + flow
    if not f32_steps or flow.dtype == torch.float32:
        return loc
    loc32 = (grid.float() + flow.float()).to(flow.dtype)
    return loc + (loc32 - loc).detach()             # exactly loc32: the two differ by less than half their size


def torch_warp(vol, flow, method='linear', fill=None, f32_steps=True):
    """SpatialTransformer (voxelmorph transform, 'ij'): vol [B, *S, C], flow [B, *S, D] -> [B, *S, C]."""
    return torch.stack([torch_interpn(vol[b], warp_loc(flow[b], f32_steps), method, fill, f32_steps) for b in range(vol.shape[0])], 0)


def resize_loc(in_shape, zoom_factor, dtype=torch.float64, device=None):
    """The resize sample grid (utils.py:256-260): tf.linspace in fp32 on every axis, then promoted."""
    D = len(in_shape)
    zf = list(zoom_factor) if isinstance(zoom_factor, (list, tuple)) else [zoom_factor] * D
    new_shape = [int(in_shape[d] * zf[d]) for d in range(D)]
    lin = [torch.from_numpy(tf_linspace_f32(0., in_shape[d] - 1., new_shape[d])).to(device) for d in range(D)]
    return torch.stack(torch.meshgrid(*lin, indexing='ij'), -1).to(dtype)


def torch_resize(x, zoom_factor, method='linear', f32_steps=True):
    """layers.Resize: x [B, *S, C] -> [B, *int(S * zoom), C]."""
    loc = resize_loc(x.shape[1:-1], zoom_factor, x.dtype, x.device)
    return torch.stack([torch_interpn(x[b], loc, method, None, f32_steps) for b in range(x.shape[0])], 0)


def torch_vec_int(vel, int_steps=7, f32_steps=True):
    """vxm VecInt (scaling and squaring, 'ij'): vel [B, *S, D]; v /= 2^steps; v += warp(v, v), steps times."""
    v = vel / (2 ** int_steps)
    for _ in range(int_steps):
        v = v + torch_warp(v, v, 'linear', None, f32_steps)
    return v


def torch_dice(y_true, y_pred, laplace=0.):
    """metrics.py:471-482, soft Dice without normalize: [B, *S, L] x2 -> [B, L]."""
    t = y_true.reshape(y_true.shape[0], -1, y_true.shape[-1])
    p = y_pred.reshape(y_pred.shape[0], -1, y_pred.shape[-1])
    top = 2 * (t * p).sum(1)
    bot = (t * t).sum(1) + (p * p).sum(1)
    if laplace > 0:
        return (top + laplace) / (bot + laplace)
    nz = bot != 0
    return torch.where(nz, top / torch.where(nz, bot, torch.ones_like(bot)), torch.zeros_like(top))


def torch_cce(y_true, y_pred, label_weights=None, sample_weight=None, from_logits=False, label_smoothing=0.,
              reduction='sum_over_batch_size'):
    """metrics.py:640-650 + the Keras categorical cross-entropy (axis -1): label weights, label smoothing,
    normalise + clip to [eps, 1 - eps] (or log_softmax), sample weights, then the reduction."""
    t = y_true
    C = y_pred.shape[-1]
    if label_weights is not None:
        t = label_weights * t
    if label_smoothing:
        t = t * (1 - label_smoothing) + label_smoothing / C
    if from_logits:
        logp = torch.log_softmax(y_pred, -1)
    else:
        eps = float(np.float32(1e-7))
        q = y_pred / y_pred.sum(-1, keepdim=True)
        logp = torch.log(torch.clamp(q, eps, float(np.float32(1) - np.float32(eps))))
    loss = -(t * logp).sum(-1)
    if sample_weight is not None:
        loss = loss * sample_weight
    if reduction == 'none':
        return loss
    return loss.sum() if reduction == 'sum' else loss.sum() / loss.numel()


def torch_local_conv3d(x, kernel, bias, kernel_size, strides=(1, 1, 1), data_format='channels_last', p0=0,
                       p_count=None):
    """LocallyConnected3D implementation 1 (layers.py:1126-1197, 1098-1099), 'valid', no activation.

    x [B, I0, I1, I2, Cin] (channels_last) or [B, Cin, I0, I1, I2]; kernel [p_count, F, Cout] with feature
    j = ((i0*k1+i1)*k2+i2)*Cin + c (channels_last) or ((c*k0+i0)*k1+i1)*k2+i2 (channels_first).
    The whole position range gives the layer's output; a range [p0, p0 + p_count) gives [B, p_count, Cout]
    (kernel and bias hold only that range).  channels_first adds the RAW reshape (1, Cout, o0, o1, o2) of the
    [o0, o1, o2, Cout] bias."""
    xl = x.permute(0, 2, 3, 4, 1) if data_format == 'channels_first' else x
    K, St = list(kernel_size), list(strides)
    win = xl.unfold(1, K[0], St[0]).unfold(2, K[1], St[1]).unfold(3, K[2], St[2])   # [B,o0,o1,o2,Cin,k0,k1,k2]
    B, O = x.shape[0], list(win.shape[1:4])
    P = O[0] * O[1] * O[2]
    if data_format == 'channels_first':
        patches = win.reshape(B, P, -1)
    else:
        patches = win.permute(0, 1, 2, 3, 5, 6, 7, 4).reshape(B, P, -1)
    if p_count is None:
        p_count = P - p0
    out = torch.einsum('bpj,pjf->bpf', patches[:, p0:p0 + p_count], kernel)
    Cout = kernel.shape[-1]
    if bias is not None:
        b = bias.reshape(-1, Cout)
        if data_format == 'channels_first':
            b = b.reshape(Cout, P).t()
        out = out + b
    if p_count != P:
        return out
    out = out.reshape([B] + O + [Cout])
    return out.permute(0, 4, 1, 2, 3) if data_format == 'channels_first' else out


# ---------------------------------------------------------------------------------------
# error bounds: (scale, k) of each gradient element
# ---------------------------------------------------------------------------------------
@torch.no_grad()
def interpn_grad_bounds(vol, loc, method, fill, gout):
    """For out = interpn(vol [*S, C], loc [*O, D]) and the upstream gradient gout [*O, C]:
    (vol_scale [*S, C], vol_k [*S, 1], loc_scale [*O, D], loc_k) of the vol and loc gradients.
    vol: scatter of w * |gout| (all w >= 0) and the number of scattered terms (+ the D roundings of w * gout);
    loc: |gout| . sum_corners (product of the other axes' weights) * |v|, 2^D * C terms (+ D)."""
    vol, loc, gout = vol.double(), loc.double(), gout.double()
    S = vol.shape[:-1]
    C, D = vol.shape[-1], loc.shape[-1]
    nvox = int(np.prod(S))
    flat = vol.reshape(nvox, C)
    keep = ~_oob(loc, S) if fill is not None else torch.ones(loc.shape[:-1], dtype=torch.bool, device=loc.device)
    keep = keep.reshape(-1)
    ag = gout.reshape(-1, C).abs() * keep[:, None]
    vs = torch.zeros((nvox, C), dtype=torch.float64, device=vol.device)
    vk = torch.zeros((nvox, 1), dtype=torch.float64, device=vol.device)
    ls = torch.zeros(loc.shape, dtype=torch.float64, device=vol.device).reshape(-1, D)
    ones = keep[:, None].double()
    strides = _strides(S)
    if method == 'linear':
        axes = _linear_axes(loc, S)
        for idx, w, bits in _corners(axes, strides):
            idx = idx.reshape(-1)
            vs.index_add_(0, idx, w.reshape(-1, 1) * ag)
            vk.index_add_(0, idx, ones)
            dot = (ag * flat[idx].abs()).sum(-1)
            for d in range(D):
                wex = torch.ones_like(dot)
                for e in range(D):
                    if e != d:
                        wex = wex * axes[e][1][bits[e]].reshape(-1)
                ls[:, d] += wex * dot
    else:
        r = [torch.clamp(torch.round(loc[..., d]).long(), 0, S[d] - 1).reshape(-1) for d in range(D)]
        idx = sum(r[d] * strides[d] for d in range(D))
        vs.index_add_(0, idx, ag)
        vk.index_add_(0, idx, ones)
    return (vs.reshape(vol.shape), vk.reshape(tuple(S) + (1,)) + D + 1,
            ls.reshape(loc.shape), (2 ** D) * C + D)


def warp_grad_bounds(vol, flow, method, fill, gout):
    """interpn_grad_bounds per batch item of a dense warp: (vol_scale, vol_k, flow_scale, flow_k)."""
    parts = [interpn_grad_bounds(vol[b], warp_loc(flow[b]), method, fill, gout[b]) for b in range(vol.shape[0])]
    return (torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]),
            torch.stack([p[2] for p in parts]), parts[0][3])


def resize_grad_bounds(x, zoom_factor, method, gout):
    """(scale, k) of the resize input gradient, x [B, *S, C]."""
    loc = resize_loc(x.shape[1:-1], zoom_factor, torch.float64, x.device)
    parts = [interpn_grad_bounds(x[b], loc, method, None, gout[b]) for b in range(x.shape[0])]
    return torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts])


@torch.no_grad()
def vec_int_grad_bounds(vel, int_steps, gout):
    """(scale, k) of the VecInt velocity gradient: the per-step bounds chained backwards.  Each step
    v' = v + warp(v, v) maps an upstream bound s to s + vol_scale(s) + flow_scale(s)."""
    vel = vel.double()
    vs = [vel / (2 ** int_steps)]
    for _ in range(int_steps):
        vs.append(vs[-1] + torch_warp(vs[-1], vs[-1]))
    s, k = gout.double().abs(), 1.0
    for v in reversed(vs[:-1]):
        a, ak, b, bk = warp_grad_bounds(v, v, 'linear', None, s)
        s = s + a + b
        k = k + float(ak.max()) + bk
    return s / (2 ** int_steps), k


@torch.no_grad()
def dice_grad_bounds(y_true, y_pred, gdice, laplace=0.):
    """Per element of d/dy_pred = a t - c p and d/dy_true = a p - c t, a = 2G/(bot+eps),
    c = 2G(top+eps)/(bot+eps)^2: (scale_pred, scale_true, k); top and bot sum V terms each."""
    t = y_true.double().reshape(y_true.shape[0], -1, y_true.shape[-1])
    p = y_pred.double().reshape(t.shape)
    G = gdice.double()
    top = 2 * (t * p).sum(1)
    bot = (t * t).sum(1) + (p * p).sum(1)
    den = bot + laplace
    live = (den != 0)
    a = torch.where(live, 2 * G.abs() / torch.where(live, den, torch.ones_like(den)), torch.zeros_like(den))[:, None]
    c = torch.where(live, 2 * G.abs() * (top + laplace) / torch.where(live, den, torch.ones_like(den)) ** 2,
                    torch.zeros_like(den))[:, None]
    sp = (a * t.abs() + c * p.abs()).reshape(y_pred.shape)
    st = (a * p.abs() + c * t.abs()).reshape(y_pred.shape)
    return sp, st, t.shape[1] + 8


@torch.no_grad()
def cce_grad_bounds(y_true, y_pred, label_weights, row_grad, from_logits=False, label_smoothing=0.):
    """(scale, k) of d/dy_pred of the cross-entropy, given row_grad = d(result) / d(per-row loss)
    (sample weight included).  Normalised: g_k = -(row_grad / s) (t_k m_k / q_k - sum_c t_c m_c);
    from_logits: g_k = row_grad (softmax_k sum_c t_c - t_k).  The row sums accumulate C terms."""
    t, p = y_true.double(), y_pred.double()
    C = p.shape[-1]
    if label_weights is not None:
        t = label_weights.double() * t
    if label_smoothing:
        t = t * (1 - label_smoothing) + label_smoothing / C
    up = row_grad.double().abs()[..., None]
    if from_logits:
        sm = torch.softmax(p, -1)
        scale = up * (sm * t.abs().sum(-1, keepdim=True) + t.abs())
        return scale, 2 * C + 8
    s = p.sum(-1, keepdim=True)
    q = p / s
    eps = float(np.float32(1e-7))
    m = (q >= eps) & (q <= float(np.float32(1) - np.float32(eps)))
    tm = torch.where(m, t.abs(), torch.zeros_like(t))
    scale = up / s.abs() * (torch.where(m, tm / torch.where(m, q, torch.ones_like(q)), torch.zeros_like(q))
                            + tm.sum(-1, keepdim=True))
    return scale, C + 8


def lc3d_grad_bounds(x, kernel, gout, kernel_size, strides, data_format='channels_last', p0=0, p_count=None):
    """(x_scale, x_k, kernel_scale, kernel_k): the same linear map applied to |x|, |kernel|, |dy|
    gives sum |dy||w| and sum |x||dy|; applied to ones it counts the terms."""
    def grads(xv, kv, gv):
        xv = xv.double().detach().requires_grad_(True)
        kv = kv.double().detach().requires_grad_(True)
        out = torch_local_conv3d(xv, kv, None, kernel_size, strides, data_format, p0, p_count)
        gx, gk = torch.autograd.grad(out, (xv, kv), gv.double())
        return gx, gk
    xs, ks = grads(x.abs(), kernel.abs(), gout.abs())
    xk, kk = grads(torch.ones_like(x), torch.ones_like(kernel), torch.ones_like(gout))
    return xs, xk + 2, ks, kk + 2
