"""
fp64 forward references of the reduction and convolution ops, and the per-element error bound of each forward
kernel.  TEST INFRASTRUCTURE (see oracle/__init__.py).

The reference graphs are the torch restatements of oracle/grad.py (Dice, CCE, LocallyConnected3D), oracle/mi.py
(soft quantisation, MI) and the ones below (Dice with normalize, hard-Dice counts, the separable convolution, MI
joint histograms and bin centres), evaluated in float64 on the fp32 inputs.  Every forward output element is held
to the bound of oracle.grad.grad_close:

    |got - ref| <= 4 * k * 2^-24 * scale + approx

  scale   the sum of the absolute values of the terms that make up the element;
  k       the fp32 rounding depth of the element: the longest run of fp32 additions / FMAs into one accumulator
          plus the roundings around it.  The *_depth helpers derive it from the launch geometry, mirroring the
          host dispatch in neurite_b200/csrc (dice_blocks, mi_blocks, the 128-voxel MMA flush, ...);
  approx  the documented error of an approximate function a kernel calls, built from the named constants below.

Hard-Dice label counts are integers and compared exactly.
"""
import numpy as np
import torch

from .grad import U, grad_close, torch_dice

F32 = np.float32

# ---------------------------------------------------------------------------------------
# documented errors of approximate functions (relative, per call)
# ---------------------------------------------------------------------------------------
EX2_APPROX_REL = 2.0 ** -22   # ex2.approx.ftz.f32 (MI soft quantisation); the PTX ISA states about 2^-22.5
EXPF_REL = 2.0 ** -22         # expf: 2 ulp (CUDA Programming Guide, mathematical functions)
LOGF_K = 2                    # logf: 1 ulp = at most 2 roundings' worth of relative error
TANHF_REL = 2.0 ** -22        # tanhf: 2 ulp
TF32_SPLIT_REL = 2.0 ** -19   # 3xTF32 product a*b ~ a_lo*b_hi + a_hi*b_lo + a_hi*b_hi: the dropped a_lo*b_lo
                              # (<= 2^-20 |ab|) and the TF32 truncation of a_lo and b_lo (<= 2^-21 |ab| each)
RCP_MUL_ROUNDINGS = 2         # CCE float4 kernel: q = p * __frcp_rn(sum p) is two roundings, not one
FTZ_ABS = 2.0 ** -126         # ex2.approx.ftz, the tensor cores and the fp32 products flush below the smallest normal
MI_ARG_ROUNDINGS = 5          # MI weight argument -alpha*log2(e) * (x - c)^2: d, d*d, the constant and the product
                              # in fp32 give a relative error of 5 roundings on the exponent E = alpha (x - c)^2,
                              # i.e. 5 * 2^-24 * E * w on the weight w = exp(-E)


def value_close(got, ref, scale, k, approx=0., what='value'):
    """grad_close for forward values."""
    grad_close(got, ref, scale, k, 4.0, what, approx)


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _cdiv(a, b):
    return -(-int(a) // int(b))


# ---------------------------------------------------------------------------------------
# Dice
# ---------------------------------------------------------------------------------------
def torch_dice_sums(y_true, y_pred, normalize=False):
    """[B, *S, L] x2 -> [B, L, 3] = (sum t p, sum t t, sum p p) (metrics.py:434-436, 471-477); normalize divides
    every voxel's label vector by its sum (divide_no_nan) first."""
    t = y_true.reshape(y_true.shape[0], -1, y_true.shape[-1])
    p = y_pred.reshape(t.shape)
    if normalize:
        def nrm(v):
            s = v.sum(-1, keepdim=True)
            return torch.where(s != 0, v / torch.where(s != 0, s, torch.ones_like(s)), torch.zeros_like(v))
        t, p = nrm(t), nrm(p)
    return torch.stack([(t * p).sum(1), (t * t).sum(1), (p * p).sum(1)], -1)


def torch_dice_fwd(y_true, y_pred, laplace=0., normalize=False):
    """soft Dice [B, L], with the reference's normalize option."""
    s = torch_dice_sums(y_true, y_pred, normalize)
    if not normalize:
        return torch_dice(y_true, y_pred, laplace)
    top, bot = 2 * s[..., 0], s[..., 1] + s[..., 2]
    if laplace > 0:
        return (top + laplace) / (bot + laplace)
    nz = bot != 0
    return torch.where(nz, top / torch.where(nz, bot, torch.ones_like(bot)), torch.zeros_like(top))


def hard_dice_counts(t_lab, p_lab, L):
    """integer label maps [B, *S] -> exact int64 counts [B, L, 3] (#t==p==l, #t==l, #p==l); labels outside [0, L)
    count nowhere (metrics.py:450-477, one_hot of an out-of-range index is all zero)."""
    t = t_lab.reshape(t_lab.shape[0], -1).long()
    p = p_lab.reshape(t.shape).long()
    out = torch.zeros((t.shape[0], L, 3), dtype=torch.int64, device=t.device)
    for b in range(t.shape[0]):
        for j, (v, m) in enumerate(((t[b], t[b] == p[b]), (t[b], None), (p[b], None))):
            keep = (v >= 0) & (v < L)
            if m is not None:
                keep = keep & m
            out[b, :, j] = torch.bincount(v[keep], minlength=L)
    return out


def dice_blocks(work_items, B, sms=None):
    """nrt_metrics.cu dice_blocks."""
    sms = sm_count() if sms is None else sms
    n = min(_cdiv(sms * 8, B), _cdiv(work_items, 4096))
    return min(max(n, 1), 2048)


def dice_sums_depth(B, nv, L, normalize=False, vec_aligned=True, sms=None):
    """k of every element of the [B, L, 3] sums nrt_dice_sums_f32 forms over nv voxels (its host dispatch):
    the longest per-thread fp32 run, the fixed-order block fold, and the fp32 rounding of the fp64 combine."""
    if not normalize and L % 4 == 0 and L // 4 <= 256 and vec_aligned:     # dice_sums_vec4_kernel<4>
        q = L // 4
        nthr = 256 // q * q
        n4 = nv * q
        nblk = dice_blocks(n4, B, sms)
        per = _cdiv(_cdiv(n4, nblk), nthr * 4) * nthr * 4
        return per // nthr + nthr // q + 1
    if not normalize and L <= 256:                                         # dice_sums_scalar_kernel
        nthr = 256 // L * L
        n = nv * L
        nblk = dice_blocks(n // 4, B, sms)
        per = _cdiv(_cdiv(n, nblk), nthr) * nthr
        return per // nthr + nthr // L + 1
    # dice_sums_voxel_kernel: every voxel of a block is added into one shared accumulator per label
    nblk = dice_blocks(nv * L // 4, B, sms)
    k = _cdiv(nv, nblk) + 1
    if normalize:
        # the label sum (a lane's serial run + 5 butterfly levels) and the division, on both factors, + product
        k += 2 * (_cdiv(L, 32) + 5 + 1) + 1
    return k


# ---------------------------------------------------------------------------------------
# categorical cross-entropy
# ---------------------------------------------------------------------------------------
_EPS32 = float(F32(1e-7))
_ONE_M_EPS32 = float(F32(1) - F32(1e-7))


def _exact_row_sum(p):
    """Rows whose fp32 sum is exact in every order and a power of two, so that the kernels' q = p / sum p is exact:
    every entry is a multiple of g, the lowest set bit of all of them, and the total is at most 2^24 g."""
    p = p.double()
    m, e = torch.frexp(p.float())
    M = (m.double() * 2 ** 24).long()
    low = (M & -M).double() * torch.ldexp(torch.ones_like(p), (e - 24).long())
    g = torch.where(p > 0, low, torch.full_like(p, np.inf)).min(-1).values
    s = p.sum(-1)
    ms, _ = torch.frexp(s)
    return torch.isfinite(g) & (s <= 2.0 ** 24 * g) & (ms == 0.5) & (p >= 0).all(-1)


@torch.no_grad()
def cce_row_bounds(y_true, y_pred, label_weights=None, sample_weight=None, from_logits=False, label_smoothing=0.,
                   vec4=False):
    """(scale, k, approx) of every per-row loss of the cross-entropy kernels, [*rows].

    Normalised: l = -sum_c t~_c log(clip(q_c)), q = p / sum p.  A relative error e of q_c is an ABSOLUTE error e
    of log q_c, whatever |log q_c| is, so the bound has two parts:
      sum_c |t~_c| |log q_c| at depth C + 7 (t~: label weight, smoothing FMA and its two constants; logf; the
        C-term dot product; the sample weight) and
      sum_c |t~_c| over the entries the normalisation reaches, at depth (C - 1) + 1 -- the C-term row sum and
        the division -- or (C - 1) + RCP_MUL_ROUNDINGS for the float4 kernel's reciprocal-then-multiply.
    An entry clipped for sure (q outside the clip range by more than that error) or a row whose sum is exact and a
    power of two (_exact_row_sum) takes no normalisation term.
    from_logits: l = -sum_c t~_c (z_c - lse), z = p - max p: sum_c |t~_c| (|z_c| + |lse|) at depth C + 7, plus
    the absolute error of lse, sum_c |t~_c| times the C-term sum's C - 1 roundings and EXPF_REL, via approx."""
    t, p = y_true.double(), y_pred.double()
    C = p.shape[-1]
    if label_weights is not None:
        t = label_weights.double() * t
    if label_smoothing:
        t = t * (1 - label_smoothing) + label_smoothing / C
    at = t.abs()
    sw = torch.ones(p.shape[:-1], dtype=torch.float64, device=p.device) if sample_weight is None \
        else sample_weight.double().expand(p.shape[:-1]).abs()
    k = C + 7
    if from_logits:
        z = p - p.max(-1, keepdim=True).values
        lse = torch.logsumexp(z, -1, keepdim=True)
        scale = (at * (z.abs() + lse.abs())).sum(-1) * sw
        approx = (4 * (C - 1) * U + EXPF_REL) * at.sum(-1) * sw
        return scale, k, approx
    q = p / p.sum(-1, keepdim=True)
    lq = torch.log(torch.clamp(q, _EPS32, _ONE_M_EPS32))
    nk = (C - 1) + (RCP_MUL_ROUNDINGS if vec4 else 1)
    e = 2 * nk * U                                     # relative error of q, with margin for the boundary test
    sure_clipped = (q < _EPS32 * (1 - e)) | (q > _ONE_M_EPS32 * (1 + e))
    reached = ~sure_clipped & ~_exact_row_sum(y_pred)[..., None]
    scale = (at * lq.abs()).sum(-1) * sw
    approx = 4 * nk * U * (at * reached).sum(-1) * sw
    return scale, k, approx


def cce_rows_per_thread(n, C, vec4, sms=None):
    """The longest per-thread run of row losses summed in fp32 by nrt_cce_f32 (its grid rule)."""
    sms = sm_count() if sms is None else sms
    cap = min(2048 * 4, sms * 8)
    if vec4:
        rpp = 256 // (C // 4) * 4
        grid = min(_cdiv(n, rpp), cap)
        return 4 * _cdiv(n, grid * rpp)
    grid = min(_cdiv(n, 256), cap)
    return _cdiv(n, grid * 256)


def cce_reduction_bound(row_scale, row_k, row_approx, ref_rows, n, C, vec4, reduction, sms=None):
    """(scale, k, approx) of the summed loss: the row bounds add up; the per-thread run, the 5-level warp sum, the
    8-warp block sum and the fp64 total's final rounding add depth on sum |row loss|; the mean divides by n once."""
    depth = cce_rows_per_thread(n, C, vec4, sms) + 5 + 8 + 1 + (1 if reduction == 'sum_over_batch_size' else 0)
    tot_rows = (4 * row_k * U * row_scale + row_approx).sum()
    scale = ref_rows.abs().sum()
    if reduction == 'sum_over_batch_size':
        tot_rows, scale = tot_rows / n, scale / n
    return scale, depth, tot_rows


# ---------------------------------------------------------------------------------------
# LocallyConnected3D
# ---------------------------------------------------------------------------------------
LC3D_ACT = {None: (None, 1.0, 0.), 'linear': (None, 1.0, 0.), 'relu': (torch.relu, 1.0, 0.),
            'sigmoid': (torch.sigmoid, 0.25, EXPF_REL + 2 * U), 'tanh': (torch.tanh, 1.0, TANHF_REL)}


@torch.no_grad()
def lc3d_fwd_bounds(x, kernel, bias, kernel_size, strides, data_format='channels_last', activation=None, p0=0,
                    p_count=None):
    """(ref, scale, k, approx) of the layer output: pre-activation scale sum |x||w| + |bias| at depth F + 7
    (a lane's FMA chain of at most F terms, the <= 5-level fold of the lanes that share a channel, the bias add,
    and one rounding of slack), times the activation's Lipschitz constant; approx: the activation's own error."""
    from .grad import torch_local_conv3d
    xd, kd = x.double(), kernel.double()
    bd = None if bias is None else bias.double()
    pre = torch_local_conv3d(xd, kd, bd, kernel_size, strides, data_format, p0, p_count)
    scale = torch_local_conv3d(xd.abs(), kd.abs(), None if bd is None else bd.abs(), kernel_size, strides,
                               data_format, p0, p_count)
    F = int(np.prod(kernel_size)) * (x.shape[1] if data_format == 'channels_first' else x.shape[-1])
    fn, lip, rel = LC3D_ACT[activation]
    ref = pre if fn is None else fn(pre)
    return ref, lip * scale, F + 7, rel * ref.abs()


# ---------------------------------------------------------------------------------------
# separable convolution
# ---------------------------------------------------------------------------------------
def same_padding(n, K, stride, dilation):
    n_out = -(-n // stride)
    total = max((n_out - 1) * stride + (K - 1) * dilation + 1 - n, 0)
    return n_out, total // 2


def torch_conv_axis(x, k, axis, padding='SAME', stride=1, dilation=1):
    """tf.nn.convolution of every feature map with the 1-D kernel k along dim `axis` (cross-correlation, zero
    'SAME' padding with the extra element at the end, or 'VALID'), in x's dtype."""
    k = torch.as_tensor(k).to(x).reshape(-1)
    n, K = x.shape[axis], k.numel()
    if padding.upper() == 'SAME':
        n_out, pb = same_padding(n, K, stride, dilation)
    else:
        n_out, pb = max(-(-(n - (K - 1) * dilation) // stride), 0), 0
    xm = torch.movedim(x, axis, 0)
    out = torch.zeros((n_out,) + tuple(xm.shape[1:]), dtype=x.dtype, device=x.device)
    o = torch.arange(n_out, device=x.device)
    for j in range(K):
        s = o * stride - pb + j * dilation
        ok = (s >= 0) & (s < n)
        if bool(ok.any()):
            out[ok] += k[j] * xm[s[ok]]
    return torch.movedim(out, 0, axis)


def torch_separable_conv(x, kernels, axes, padding='SAME', strides=None, dilations=None):
    """utils.separable_conv (batched): one pass per axis of the [B, *space, C] tensor x."""
    strides = strides or [1] * len(axes)
    dilations = dilations or [1] * len(axes)
    for ax, k, s, d in zip(axes, kernels, strides, dilations):
        x = torch_conv_axis(x, k, ax + 1, padding, s, d)
    return x


def sepconv_bounds(x, kernels, axes, padding='SAME', strides=None, dilations=None):
    """(scale, k): the same passes with |kernel| on |x| bound every propagated error; each pass adds its K taps
    (one FMA each) to the depth."""
    scale = torch_separable_conv(x.double().abs(), [torch.as_tensor(k).double().abs() for k in kernels], axes,
                                 padding, strides, dilations)
    return scale, sum(int(torch.as_tensor(k).numel()) for k in kernels) + len(axes)


# ---------------------------------------------------------------------------------------
# MutualInformation: bin centres, joint histograms
# ---------------------------------------------------------------------------------------
def mi_centers_f32(x, nb):
    """mi_centers_kernel on the fp32 min / max of x: delta = (mx - mn) / (nb - 1), c_i = mn + delta * i, each
    operation one fp32 rounding, the ends pinned to mn and mx.  numpy fp32 [nb]."""
    x = np.asarray(x, F32)
    mn, mx = F32(x.min()), F32(x.max())
    c = np.empty(nb, F32)
    if nb == 1:
        c[0] = mn
        return c
    delta = F32(F32(mx - mn) / F32(nb - 1))
    c[:] = F32(mn) + F32(delta * np.arange(nb, dtype=F32))
    c[0], c[-1] = mn, mx
    return c


def mi_blocks(nv, items, sms=None, per_sm=None):
    """nrt_mi.cu mi_blocks (NRT_MI_CTAS_PER_SM: per_sm)."""
    sms = sm_count() if sms is None else sms
    per_sm = per_sm if per_sm and per_sm > 0 else 4
    n = min(_cdiv(sms * per_sm, items), _cdiv(nv, 1024))
    return min(max(n, 1), 592)


def mi_hist_depth(nv, items, nbx, nby, generic, spc, sms=None, per_sm=None):
    """(k of each joint-histogram element, k of each marginal).
    Tensor-core kernel: a warp takes ceil(chunks / (nblk * 8)) chunks of 8*spc voxels; an accumulator run is 128
    voxels (16 steps x 3 MMAs, each adding 8 products: <= 16*3 + 8 roundings), flushed into a per-lane fp32
    total once per run; then the 8-warp fold and the fp64 combine.  Marginals: two roundings per step (pair sum
    and accumulate), the 2-level lane shuffle, the 8-warp fold, the combine.
    CUDA-core kernel: one FMA chain per block over ceil(nv / 32 / nblk) 32-voxel chunks; marginals likewise."""
    nblk = mi_blocks(nv, items, sms, per_sm)
    if generic:
        vox = _cdiv(_cdiv(nv, 32), nblk) * 32
        return vox + 1, vox + 1
    ch = 8 * spc
    chunks = _cdiv(_cdiv(nv, ch), nblk * 8)
    steps = chunks * spc
    k_h = (16 * 3 + 8) + _cdiv(steps, 16) + 1 + 8 + 1
    k_m = 2 * steps + 2 + 8 + 1
    return k_h, k_m


@torch.no_grad()
def mi_weights(v, quant, centers, alpha, lo, hi):
    """fp64 soft-quantisation weights of one operand [items, nv, nb] (quant: v [items, nv] intensities; else v is
    the map itself) and the per-weight approx error (MI_ARG_ROUNDINGS on the exponent + the exp itself)."""
    if not quant:
        return v.double(), torch.zeros_like(v, dtype=torch.float64)
    c = torch.as_tensor(centers, dtype=torch.float64, device=v.device)
    xc = torch.clamp(v.double(), float(F32(lo)), float(F32(hi)))[..., None]
    E = float(F32(alpha)) * (xc - c) ** 2
    w = torch.exp(-E)
    return w, w * (MI_ARG_ROUNDINGS * U * E + EX2_APPROX_REL)


@torch.no_grad()
def mi_hist_reference(wx, ex, wy, ey, tensor_cores):
    """fp64 stats [items, nbx*nby + nbx + nby] = (joint histogram row-major, x marginal, y marginal) and the
    approx term of each element: the weights' errors carried through the products, plus TF32_SPLIT_REL per
    product on the tensor-core path, plus FTZ_ABS for each of the two weights and the product of every voxel."""
    nv = wx.shape[1]
    h = torch.einsum('bvi,bvj->bij', wx, wy)
    ah = torch.einsum('bvi,bvj->bij', ex, wy) + torch.einsum('bvi,bvj->bij', wx, ey) + 3 * nv * FTZ_ABS
    if tensor_cores:
        ah = ah + TF32_SPLIT_REL * h
    n = wx.shape[0]
    stats = torch.cat([h.reshape(n, -1), wx.sum(1), wy.sum(1)], 1)
    approx = torch.cat([ah.reshape(n, -1), ex.sum(1) + nv * FTZ_ABS, ey.sum(1) + nv * FTZ_ABS], 1)
    return stats, approx


def mi_from_stats(stats, nbx, nby, eps=1e-7):
    """metrics.py:265-292 on fp64 sums [items, PS] -> [items]."""
    npair = nbx * nby
    h, sx, sy = stats[:, :npair].reshape(-1, nbx, nby), stats[:, npair:npair + nbx], stats[:, npair + nbx:]
    pxy = h / (h.sum((1, 2), keepdim=True) + eps)
    px = sx / (sx.sum(1, keepdim=True) + eps)
    py = sy / (sy.sum(1, keepdim=True) + eps)
    pxpy = px[:, :, None] * py[:, None, :]
    return (pxy * torch.log(pxy / (pxpy + eps) + eps)).sum((1, 2))

