"""
neurite_b200.utils -- drop-in for the interpolation part of neurite.utils
(adalca/neurite: neurite/tf/utils/utils.py), on torch CUDA tensors, channels-last.

    interpn(vol, loc, interp_method='linear', fill_value=None)     utils.py:73-220
    resize(vol, zoom_factor, interp_method='linear') / zoom        utils.py:223-265
    transform(vol, loc_shift, interp_method, indexing, fill_value) voxelmorph.utils.transform contract
    sub2ind2d, prod_n, ndgrid, meshgrid, volshape_to_ndgrid, volshape_to_meshgrid,
    batch_channel_flatten, flatten_axes                            utils.py:333-476, 1068-1226

Same names, argument order, defaults and exception classes as the reference.  The
arithmetic runs in the hand-written CUDA kernels behind the C ABI (include/neurite_b200.h);
the helpers that only build index grids stay thin torch code for API parity -- the fused
kernels never materialise them.
"""
import numpy as np
import torch

from . import _lib
from ._lib import lib, check, ptr, stream_ptr, i32_array, method_id, require_cuda

MAX_DIMS = 3             # warp / resize (the layers that call them are 1-3 D)
MAX_INTERPN_DIMS = 5     # interpn itself takes any D in the reference (utils.py:106-120); built for 1..5


def _as_f32(t):
    return t if t.dtype == torch.float32 else t.to(torch.float32)


# ---------------------------------------------------------------------------------------
# interpn
# ---------------------------------------------------------------------------------------
def interpn(vol, loc, interp_method='linear', fill_value=None):
    """N-D gridded interpolation (reference utils.py:73-220).

    vol: [*vol_shape] or [*vol_shape, C]; loc: list of D tensors or a [*new_shape, D] tensor.
    Edge-clamped ('nearest' extrapolation) unless fill_value is given."""
    if isinstance(loc, (list, tuple)):
        loc = torch.stack(list(loc), -1)                                # :106-107
    nb_dims = loc.shape[-1]
    input_vol_ndim = vol.dim()
    if vol.dim() not in [nb_dims, nb_dims + 1]:                         # :111-113
        raise Exception("Number of loc Tensors %d does not match volume dimension %d"
                        % (nb_dims, len(vol.shape[:-1])))
    if nb_dims > vol.dim():                                             # :115-117
        raise Exception("Loc dimension %d does not match volume dimension %d" % (nb_dims, vol.dim()))
    method = method_id(interp_method)                                   # AssertionError, :194-195
    if nb_dims > MAX_INTERPN_DIMS:
        raise NotImplementedError('neurite_b200.interpn supports up to %d spatial dims (got %d)'
                                  % (MAX_INTERPN_DIMS, nb_dims))
    require_cuda(vol, loc)
    if vol.dim() == nb_dims:                                            # :119-120
        vol = vol.unsqueeze(-1)
    out_dtype = vol.dtype
    if not vol.dtype.is_floating_point and method == _lib.NRT_LINEAR:
        raise TypeError('linear interpolation needs a floating-point volume (reference: dtype error in wt * vol_val)')
    vol32 = _as_f32(vol).contiguous()
    loc32 = _as_f32(loc).contiguous()                                   # :123-127
    if torch.is_grad_enabled() and (vol32.requires_grad or loc32.requires_grad):
        if nb_dims > MAX_DIMS:
            raise NotImplementedError('interpn gradients are built for up to %d spatial dims' % MAX_DIMS)
        out = _InterpnFn.apply(vol32, loc32, method, fill_value)
    else:
        out = _interpn_raw(vol32, loc32, method, fill_value)
    if out.dtype != out_dtype:
        out = out.to(out_dtype)
    if input_vol_ndim == nb_dims:                                       # :216-218
        out = out[..., 0]
    return out


def _interpn_raw(vol32, loc32, method, fill_value):
    nb_dims = loc32.shape[-1]
    C = vol32.shape[-1]
    out_shape = tuple(loc32.shape[:-1])
    n_out = int(np.prod(out_shape)) if len(out_shape) else 1
    out = torch.empty(out_shape + (C,), dtype=torch.float32, device=vol32.device)
    if out.numel() == 0:
        return out
    if nb_dims == 3 and out_shape == tuple(vol32.shape[:-1]):
        # the sample grid has the volume's own shape (what transform() passes): tiled fast path
        with torch.cuda.device(vol32.device):
            check(lib.nrt_interpn_grid_f32(ptr(vol32), ptr(loc32), ptr(out), i32_array(vol32.shape[:-1]), C, method,
                                           0 if fill_value is None else 1,
                                           0.0 if fill_value is None else float(fill_value), 0,
                                           stream_ptr(vol32.device)))
        return out
    with torch.cuda.device(vol32.device):
        check(lib.nrt_interpn_f32(ptr(vol32), i32_array(vol32.shape[:-1]), nb_dims, C, ptr(loc32), n_out, method,
                                  0 if fill_value is None else 1, 0.0 if fill_value is None else float(fill_value),
                                  ptr(out), stream_ptr(vol32.device)))
    return out


class _InterpnFn(torch.autograd.Function):
    """autograd shell around nrt_interpn_f32 / nrt_interpn_bwd_f32 (TF autodiff semantics)."""

    @staticmethod
    def forward(ctx, vol32, loc32, method, fill_value):
        ctx.save_for_backward(vol32, loc32)
        ctx.method, ctx.fill = method, fill_value
        return _interpn_raw(vol32.detach(), loc32.detach(), method, fill_value)

    @staticmethod
    def backward(ctx, g):
        vol32, loc32 = ctx.saved_tensors
        g = g.contiguous().to(torch.float32)
        D, C = loc32.shape[-1], vol32.shape[-1]
        gvol = torch.zeros_like(vol32) if ctx.needs_input_grad[0] else None
        gloc = torch.empty_like(loc32) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(vol32.device):
            check(lib.nrt_interpn_bwd_f32(ptr(vol32), i32_array(vol32.shape[:-1]), D, C, ptr(loc32),
                                          loc32.numel() // D, ctx.method, 0 if ctx.fill is None else 1, ptr(g),
                                          ptr(gvol), ptr(gloc), stream_ptr(vol32.device)))
        return gvol, gloc, None, None


# ---------------------------------------------------------------------------------------
# resize / zoom
# ---------------------------------------------------------------------------------------
def _resize_batched(x, zoom_factor, interp_method, out_z0=0, out_n0=None):
    """x [B,*S,C] -> [B,*int(S*zoom),C] (one launch for the whole batch)."""
    method = method_id(interp_method)
    require_cuda(x)
    ndims = x.dim() - 2
    if ndims > MAX_DIMS:
        raise NotImplementedError('resize supports up to %d spatial dims' % MAX_DIMS)
    in_shape = [int(s) for s in x.shape[1:-1]]
    new_shape = [int(in_shape[f] * zoom_factor[f]) for f in range(ndims)]   # :256-257
    x32 = _as_f32(x).contiguous()
    if out_n0 is None:
        out_n0 = new_shape[0]
    if torch.is_grad_enabled() and x32.requires_grad:
        if out_z0 != 0 or out_n0 != new_shape[0]:
            raise NotImplementedError('gradients are built for whole-volume resize only')
        out = _ResizeFn.apply(x32, tuple(in_shape), tuple(new_shape), method)
    else:
        out = _resize_raw(x32, in_shape, new_shape, method, out_z0, out_n0)
    return out if x.dtype == torch.float32 else out.to(x.dtype)


def _resize_raw(x32, in_shape, new_shape, method, out_z0, out_n0):
    B, C = x32.shape[0], x32.shape[-1]
    ndims = len(in_shape)
    out = torch.empty((B, out_n0) + tuple(new_shape[1:]) + (C,), dtype=torch.float32, device=x32.device)
    if out.numel():
        with torch.cuda.device(x32.device):
            check(lib.nrt_resize_f32(ptr(x32), ptr(out), B, i32_array(in_shape), i32_array(new_shape), ndims, C,
                                     method, out_z0, out_n0, stream_ptr(x32.device)))
    return out


class _ResizeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x32, in_shape, new_shape, method):
        ctx.in_shape, ctx.new_shape, ctx.method, ctx.xshape = in_shape, new_shape, method, tuple(x32.shape)
        return _resize_raw(x32.detach(), in_shape, new_shape, method, 0, new_shape[0])

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous().to(torch.float32)
        gx = torch.zeros(ctx.xshape, dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            check(lib.nrt_resize_bwd_f32(ptr(g), ptr(gx), ctx.xshape[0], i32_array(ctx.in_shape), i32_array(ctx.new_shape),
                                         len(ctx.in_shape), ctx.xshape[-1], ctx.method, stream_ptr(g.device)))
        return gx, None, None, None


def resize(vol, zoom_factor, interp_method='linear'):
    """reference utils.py:223-265: zoom a single volume [*S, C] (or [*S] with a zoom list)."""
    if isinstance(zoom_factor, (list, tuple)):
        ndims = len(zoom_factor)
        vol_shape = vol.shape[:ndims]
        assert len(vol_shape) in (ndims, ndims + 1), \
            "zoom_factor length %d does not match ndims %d" % (len(vol_shape), ndims)      # :241-242
        zoom_factor = list(zoom_factor)
    else:
        vol_shape = vol.shape[:-1]
        ndims = len(vol_shape)
        zoom_factor = [zoom_factor] * ndims
    if all(z == 1 for z in zoom_factor):                                 # :250-251
        return vol
    squeeze = vol.dim() == ndims
    v = vol.unsqueeze(-1) if squeeze else vol
    out = _resize_batched(v.unsqueeze(0), zoom_factor, interp_method)[0]
    return out[..., 0] if squeeze else out


zoom = resize


# ---------------------------------------------------------------------------------------
# dense warp (voxelmorph.utils.transform contract, SURVEY.md 8c)
# ---------------------------------------------------------------------------------------
def _warp_batched(vol, flow, interp_method='linear', fill_value=None, halo=0,
                  src_z0=0, full_s0=None, out_z0=0, err_flag=None):
    """vol [B, src_n0, *S_rest, C], flow [B, out_n0, *S_rest, D] -> [B, out_n0, *S_rest, C].

    With the defaults this is the whole-volume warp; the slab arguments are used by
    neurite_b200.dist for z-slab sharding (vol holds planes [src_z0, src_z0+src_n0) of a
    volume of full extent full_s0; flow/out are planes [out_z0, out_z0+out_n0))."""
    method = method_id(interp_method)
    require_cuda(vol, flow)
    D = flow.shape[-1]
    if vol.dim() != D + 2 or flow.dim() != D + 2:
        raise Exception("Number of loc Tensors %d does not match volume dimension %d" % (D, vol.dim() - 2))
    if D > MAX_DIMS:
        raise NotImplementedError('warp supports up to %d spatial dims' % MAX_DIMS)
    if not vol.dtype.is_floating_point and method == _lib.NRT_LINEAR:
        raise TypeError('linear interpolation needs a floating-point volume')
    vol32 = _as_f32(vol).contiguous()
    flow32 = _as_f32(flow).contiguous()
    B, C = vol32.shape[0], vol32.shape[-1]
    src_n0, out_n0 = vol32.shape[1], flow32.shape[1]
    if full_s0 is None:
        full_s0 = src_n0
    if tuple(vol32.shape[2:-1]) != tuple(flow32.shape[2:-1]) or flow32.shape[0] != B:
        raise ValueError('vol %s and flow %s disagree on batch / trailing spatial dims'
                         % (tuple(vol.shape), tuple(flow.shape)))
    shape = [int(full_s0)] + [int(s) for s in vol32.shape[2:-1]]
    slab = (int(src_z0), int(src_n0), int(out_z0), int(out_n0))
    if torch.is_grad_enabled() and (vol32.requires_grad or flow32.requires_grad):
        if slab != (0, shape[0], 0, shape[0]):
            raise NotImplementedError('gradients are built for whole-volume warps only')
        out = _WarpFn.apply(vol32, flow32, tuple(shape), method, fill_value, int(halo))
    else:
        out = _warp_raw(vol32, flow32, shape, method, fill_value, slab, int(halo), err_flag)
    return out if vol.dtype == torch.float32 else out.to(vol.dtype)


def _warp_raw(vol32, flow32, shape, method, fill_value, slab, halo, err_flag):
    B, C, D = vol32.shape[0], vol32.shape[-1], flow32.shape[-1]
    out = torch.empty(tuple(flow32.shape[:-1]) + (C,), dtype=torch.float32, device=vol32.device)
    if out.numel():
        with torch.cuda.device(vol32.device):
            check(lib.nrt_warp_f32(ptr(vol32), ptr(flow32), ptr(out), B, i32_array(shape), D, C, method,
                                   0 if fill_value is None else 1, 0.0 if fill_value is None else float(fill_value),
                                   slab[0], slab[1], slab[2], slab[3], halo, ptr(err_flag), stream_ptr(vol32.device)))
    return out


def _inner_contiguous(t):
    """True if every batch item of t [B, ...] is a dense block (only the batch stride may be larger)."""
    exp = 1
    for size, stride in zip(reversed(t.shape[1:]), reversed(t.stride()[1:])):
        if size != 1 and stride != exp:
            return False
        exp *= size
    return t.shape[0] <= 1 or t.stride(0) >= exp


def _warp_views(vol_v, flow_v, out_v, full_s0, method, fill_value, src_z0, out_z0, halo=0, err_flag=None):
    """Warp into a caller-owned output: vol_v [B, src_n0, H, W, C], flow_v [B, out_n0, H, W, 3], out_v
    [B, out_n0, H, W, C] may be PLANE SUB-RANGES of larger [B, planes, ...] buffers (dense inside a batch item,
    strided across the batch) -- nrt_warp_strided_f32.  No allocation, no synchronisation."""
    require_cuda(vol_v, flow_v, out_v)
    for v in (vol_v, flow_v, out_v):
        if v.dtype != torch.float32 or not _inner_contiguous(v):
            raise ValueError('_warp_views needs fp32 views that are dense inside each batch item')
    B, C, D = vol_v.shape[0], vol_v.shape[-1], flow_v.shape[-1]
    if out_v.numel() == 0:
        return out_v
    shape = [int(full_s0)] + [int(s) for s in vol_v.shape[2:-1]]
    bs = lambda v: int(v.stride(0)) if v.shape[0] > 1 else 0          # noqa: E731
    with torch.cuda.device(vol_v.device):
        check(lib.nrt_warp_strided_f32(ptr(vol_v), ptr(flow_v), ptr(out_v), B, i32_array(shape), D, C, method,
                                       0 if fill_value is None else 1, 0.0 if fill_value is None else float(fill_value),
                                       int(src_z0), int(vol_v.shape[1]), int(out_z0), int(out_v.shape[1]), int(halo),
                                       ptr(err_flag), bs(vol_v), bs(flow_v), bs(out_v), stream_ptr(vol_v.device)))
    return out_v


class _WarpFn(torch.autograd.Function):
    """autograd shell around nrt_warp_f32 / nrt_warp_bwd_f32."""

    @staticmethod
    def forward(ctx, vol32, flow32, shape, method, fill_value, halo):
        ctx.save_for_backward(vol32, flow32)
        ctx.shape, ctx.method, ctx.fill = shape, method, fill_value
        return _warp_raw(vol32.detach(), flow32.detach(), list(shape), method, fill_value,
                         (0, shape[0], 0, shape[0]), halo, None)

    @staticmethod
    def backward(ctx, g):
        vol32, flow32 = ctx.saved_tensors
        g = g.contiguous().to(torch.float32)
        gvol = torch.zeros_like(vol32) if ctx.needs_input_grad[0] else None
        gflow = torch.empty_like(flow32) if ctx.needs_input_grad[1] else None
        with torch.cuda.device(vol32.device):
            check(lib.nrt_warp_bwd_f32(ptr(vol32), ptr(flow32), ptr(g), ptr(gvol), ptr(gflow), vol32.shape[0],
                                       i32_array(ctx.shape), flow32.shape[-1], vol32.shape[-1], ctx.method,
                                       0 if ctx.fill is None else 1, stream_ptr(vol32.device)))
        return gvol, gflow, None, None, None, None


_HOST_STREAMS = {}


def warp_host(vol, flow, out=None, interp_method='linear', fill_value=None, halo=0, device=None, chunk=1):
    """Dense warp for HOST tensors: vol [B,*S,C], flow [B,*S,D] on the CPU (pinned memory
    for full PCIe speed) -> out [B,*S,C] on the CPU (written in place if given).

    The batch is cut into chunks of `chunk` volumes that travel over three CUDA streams in
    a ring: the host->device copy of chunk i+1 overlaps the kernel and the device->host copy
    of chunk i (the two PCIe directions are independent), so a batch costs about
    max(H2D, D2H) instead of H2D + kernel + D2H.  Returns after the result is in `out`."""
    method = method_id(interp_method)
    if vol.is_cuda or flow.is_cuda:
        raise ValueError('warp_host takes CPU tensors; use SpatialTransformer / transform for device tensors')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    vol = vol.to(torch.float32).contiguous()
    flow = flow.to(torch.float32).contiguous()
    B = vol.shape[0]
    if out is None:
        out = torch.empty(tuple(flow.shape[:-1]) + (vol.shape[-1],), dtype=torch.float32, pin_memory=True)
    key = (dev.type, dev.index)
    if key not in _HOST_STREAMS:
        _HOST_STREAMS[key] = [torch.cuda.Stream(device=dev) for _ in range(3)]
    streams = _HOST_STREAMS[key]
    cur = torch.cuda.current_stream(dev)
    shape = [int(s) for s in vol.shape[1:-1]]
    done = []
    for i, b0 in enumerate(range(0, B, chunk)):
        st = streams[i % len(streams)]
        st.wait_stream(cur)
        with torch.cuda.stream(st):
            dv = vol[b0:b0 + chunk].to(dev, non_blocking=True)
            df = flow[b0:b0 + chunk].to(dev, non_blocking=True)
            o = _warp_raw(dv, df, shape, method, fill_value, (0, shape[0], 0, shape[0]), int(halo), None)
            out[b0:b0 + chunk].copy_(o, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(st)
            done.append(ev)
    for ev in done:
        ev.synchronize()
    return out


def transform(vol, loc_shift, interp_method='linear', indexing='ij', fill_value=None):
    """voxelmorph.utils.transform: interpn(vol, ndgrid + loc_shift).  vol [*S, C], shift [*S, D]."""
    if indexing not in ('ij', 'xy'):
        raise ValueError("indexing parameter must be either 'xy' or 'ij'")
    if indexing == 'xy' and loc_shift.shape[-1] > 1:
        # meshgrid 'xy' swaps which axis carries grid 0/1 (utils.py:460-464); equivalent to
        # adding the transposed identity grid -- rarely used, so go through interpn directly
        mesh = volshape_to_meshgrid(loc_shift.shape[:-1], indexing='xy', device=loc_shift.device)
        loc = [mesh[d].to(torch.float32) + loc_shift[..., d] for d in range(loc_shift.shape[-1])]
        return interpn(vol, loc, interp_method=interp_method, fill_value=fill_value)
    squeeze = vol.dim() == loc_shift.shape[-1]
    v = vol.unsqueeze(-1) if squeeze else vol
    out = _warp_batched(v.unsqueeze(0), loc_shift.unsqueeze(0), interp_method, fill_value)[0]
    return out[..., 0] if squeeze else out


# ---------------------------------------------------------------------------------------
# thin helpers kept for API parity (the kernels fuse them away)
# ---------------------------------------------------------------------------------------
def sub2ind2d(siz, subs, **kwargs):
    """utils.py:1068-1082 (row-major despite the reference docstring)."""
    assert len(siz) == len(subs), 'found inconsistent siz and subs: %d %d' % (len(siz), len(subs))
    k = np.cumprod(siz[::-1])
    ndx = subs[-1]
    for i, v in enumerate(subs[:-1][::-1]):
        ndx = ndx + v * int(k[i])
    return ndx


def prod_n(lst):
    """utils.py:1085-1092."""
    prod = lst[0]
    for p in lst[1:]:
        prod = prod * p
    return prod


def meshgrid(*args, **kwargs):
    """utils.py:398-476."""
    indexing = kwargs.pop('indexing', 'xy')
    if kwargs:
        key = list(kwargs.keys())[0]
        raise TypeError("'{}' is an invalid keyword argument for this function".format(key))
    if indexing not in ('xy', 'ij'):
        raise ValueError("indexing parameter must be either 'xy' or 'ij'")
    args = [torch.as_tensor(a) for a in args]
    return list(torch.meshgrid(*args, indexing=indexing))


def ndgrid(*args, **kwargs):
    """utils.py:382-395."""
    return meshgrid(*args, indexing='ij', **kwargs)


def volshape_to_ndgrid(volshape, device=None, **kwargs):
    """utils.py:333-353."""
    if not all(float(d).is_integer() for d in volshape):
        raise ValueError("volshape needs to be a list of integers")
    return ndgrid(*[torch.arange(0, int(d), device=device) for d in volshape], **kwargs)


def volshape_to_meshgrid(volshape, device=None, **kwargs):
    """utils.py:356-379."""
    if not all(float(d).is_integer() for d in volshape):
        raise ValueError("volshape needs to be a list of integers")
    return meshgrid(*[torch.arange(0, int(d), device=device) for d in volshape], **kwargs)


def flatten_axes(x, axes):
    """utils.py:1195-1226."""
    assert isinstance(axes, (list, tuple, range)), 'axes must be list or tuple of axes to be flattened'
    assert np.all(np.diff(axes) == 1), 'axes need to be contiguous'
    if axes[0] < 0:
        assert axes[-1] < 0, 'if one axis is negative, all have to be negative'
    assert axes[-1] < x.dim(), 'axis %d outside max axis %d' % (axes[-1], x.dim() - 1)
    shp = list(x.shape)
    new = shp[:axes[0]] + [-1]
    if axes[-1] < x.dim() - 1 and not (axes[-1] == -1):
        new += shp[axes[-1] + 1:]
    return x.reshape(new)


def batch_channel_flatten(x):
    """utils.py:1175-1188."""
    return flatten_axes(x, range(1, x.dim() - 1))


flatten_batch_channel = batch_channel_flatten


# ---------------------------------------------------------------------------------------
# soft quantisation (utils.py:1095-1172) -- the tensor op; MutualInformation fuses it (metrics.py)
# ---------------------------------------------------------------------------------------
_SCRATCH = {}


def _stream_scratch(cache, max_streams, device, nbytes):
    """Scratch buffer per (device, stream), LRU-bounded to `max_streams` entries (dicts keep insertion order)."""
    key = (device.type, device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = cache.pop(key, None)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
    cache[key] = buf                                   # most recently used last
    while len(cache) > max_streams:
        cache.pop(next(iter(cache)))
    return buf


def _scratch(device, nbytes):
    return _stream_scratch(_SCRATCH, 8, device, nbytes)


def _item_stats(x2d, kind):
    """Per-row reduction of the contiguous fp32 [items, n] view x2d on the device (nrt_item_stats_f32): [items] for
    NRT_STAT_SD / MAX / ABSMAX, [items, 2] = (min, max) for NRT_STAT_MINMAX."""
    items, n = x2d.shape
    out = torch.empty((items, 2) if kind == _lib.NRT_STAT_MINMAX else (items,), dtype=torch.float32, device=x2d.device)
    nb = lib.nrt_item_stats_workspace_bytes(int(items), int(n))
    ws = _scratch(x2d.device, nb)
    with torch.cuda.device(x2d.device):
        check(lib.nrt_item_stats_f32(ptr(x2d), int(items), int(n), int(kind), ptr(out), ptr(ws), nb,
                                     stream_ptr(x2d.device)))
    return out


def minmax(x, group=None):
    """device tensor [min(x), max(x)] (K.min / K.max, utils.py:1151-1152), no host sync.
    With `group`, the extrema over every rank's shard (one MIN all-reduce of [min, -max])."""
    require_cuda(x)
    out = _item_stats(_as_f32(x).contiguous().reshape(1, -1), _lib.NRT_STAT_MINMAX).reshape(2)
    if group is not None:
        import torch.distributed as dist
        packed = torch.stack([out[0], -out[1]])
        dist.all_reduce(packed, op=dist.ReduceOp.MIN, group=group)
        out = torch.stack([packed[0], -packed[1]])
    return out


def bin_centers_from_range(mm, nb_bins):
    """tf.linspace(min, max, nb_bins) in fp32 on the device (utils.py:1153)."""
    centers = torch.empty(int(nb_bins), dtype=torch.float32, device=mm.device)
    with torch.cuda.device(mm.device):
        check(lib.nrt_mi_bin_centers_f32(ptr(mm), int(nb_bins), ptr(centers), stream_ptr(mm.device)))
    return centers


def soft_quantize(x, bin_centers=None, nb_bins=16, alpha=1, min_clip=-np.inf, max_clip=np.inf,
                  return_log=False):
    """(Softly) quantize intensities with RBFs, utils.py:1099-1172: [...] -> [..., B]."""
    require_cuda(x)
    x32 = _as_f32(x).contiguous()
    if bin_centers is not None:
        centers = torch.as_tensor(bin_centers, dtype=torch.float32, device=x.device).contiguous()
        assert nb_bins is None, 'cannot provide both bin_centers and nb_bins'
        nb_bins = centers.shape[0]
    else:
        if nb_bins is None:
            nb_bins = 16
        centers = bin_centers_from_range(minmax(x32), nb_bins)
    out = torch.empty(tuple(x32.shape) + (int(nb_bins),), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.nrt_soft_quantize_f32(ptr(x32), x32.numel(), ptr(centers), int(nb_bins), float(alpha),
                                        float(min_clip), float(max_clip), int(bool(return_log)), ptr(out),
                                        stream_ptr(x.device)))
    return out


soft_digitize = soft_quantize


# ---------------------------------------------------------------------------------------
# gaussian_kernel / separable_conv / subsample_axis (utils.py:581-826)
# ---------------------------------------------------------------------------------------
def gaussian_kernel(sigma, windowsize=None, indexing='ij', separate=False, random=False, min_sigma=0,
                    dtype=torch.float32, seed=None, device=None):
    """N-D Gaussian kernel, utils.py:581-662.  Returns torch tensors (on `device`, default CPU);
    built on the host in fp32 with the reference's operation order.  `random=True` draws each
    SD uniformly from [min_sigma, sigma) with a torch generator (TF's stream is not reproducible
    elsewhere)."""
    assert dtype.is_floating_point, f'{dtype} is not a real floating-point type'
    npdt = {torch.float32: np.float32, torch.float64: np.float64, torch.float16: np.float16}[dtype]
    if not isinstance(sigma, (list, tuple)):
        sigma = [sigma]
    if not isinstance(min_sigma, (list, tuple)):
        min_sigma = [min_sigma] * len(sigma)
    eps = np.finfo(npdt).eps
    sigma = [max(f, eps) for f in sigma]
    min_sigma = [max(f, eps) for f in min_sigma]
    if windowsize is None:
        windowsize = [np.round(f * 3) * 2 + 1 for f in sigma]
    if not isinstance(windowsize, (list, tuple)):
        windowsize = [windowsize]
    if len(sigma) != len(windowsize):
        raise ValueError(f'sigma {sigma} and width {windowsize} differ in length')
    center = [(w - 1) / 2 for w in windowsize]
    mesh = [np.arange(w) - c for w, c in zip(windowsize, center)]
    mesh = [-0.5 * x**2 for x in mesh]
    if not separate:
        mesh = np.meshgrid(*mesh, indexing=indexing)
    mesh = [m.astype(npdt) for m in mesh]
    if random:
        gen = torch.Generator().manual_seed(int(np.random.default_rng(seed).integers(2**31)))
        sigma = [float(a + (b - a) * torch.rand(1, generator=gen).item()) for a, b in zip(min_sigma, sigma)]
    exponent = [m / npdt(s**2) for m, s in zip(mesh, sigma)]
    if not separate:
        exponent = [np.sum(np.stack(exponent), axis=0, dtype=np.float64).astype(npdt)]
    kernel = [np.exp(x) for x in exponent]
    kernel = [x / np.sum(x, dtype=np.float64).astype(npdt) for x in kernel]
    kernel = [torch.as_tensor(k, dtype=dtype, device=device) for k in kernel]
    return kernel if len(kernel) > 1 else kernel[0]


def _same_padding(n, k, stride, dilation):
    n_out = -(-n // stride)
    total = max((n_out - 1) * stride + (k - 1) * dilation + 1 - n, 0)
    return n_out, total // 2


def _conv_axis_raw(x32, kdev, axis, stride, dilation, pad_before, n_out):
    """one nrt_sepconv_axis_f32 pass along dim `axis` of a contiguous fp32 tensor."""
    shp = list(x32.shape)
    outer = int(np.prod(shp[:axis], dtype=np.int64))
    L = shp[axis]
    inner = int(np.prod(shp[axis + 1:], dtype=np.int64))
    out = torch.empty(shp[:axis] + [int(n_out)] + shp[axis + 1:], dtype=torch.float32, device=x32.device)
    with torch.cuda.device(x32.device):
        check(lib.nrt_sepconv_axis_f32(ptr(x32), ptr(out), outer, L, inner, ptr(kdev), int(kdev.numel()), int(stride),
                                       int(dilation), int(pad_before), int(n_out), stream_ptr(x32.device)))
    return out


class _ConvAxisFn(torch.autograd.Function):
    """autograd shell of one pass: d/dx of a stride-1 cross-correlation is the correlation of the
    upstream gradient with the flipped kernel and the complementary padding."""

    @staticmethod
    def forward(ctx, x, kdev, axis, stride, dilation, pad_before, n_out):
        x32 = _as_f32(x.detach()).contiguous()
        ctx.save_for_backward(kdev)
        ctx.cfg = (axis, stride, dilation, pad_before, x32.shape[axis])
        return _conv_axis_raw(x32, kdev, axis, stride, dilation, pad_before, n_out)

    @staticmethod
    def backward(ctx, g):
        (kdev,) = ctx.saved_tensors
        axis, stride, dilation, pad_before, L = ctx.cfg
        if stride != 1:
            raise NotImplementedError('gradient of a strided separable_conv pass')
        K = kdev.numel()
        gx = _conv_axis_raw(_as_f32(g).contiguous(), kdev.flip(0).contiguous(), axis, 1, dilation,
                            (K - 1) * dilation - pad_before, L)
        return gx, None, None, None, None, None, None


def separable_conv(x, kernels, axis=None, batched=False, padding='SAME', strides=None, dilations=None):
    """Apply 1-D kernels along axes of a tensor with a trailing feature dimension; the same
    filters across features (utils.py:665-751).  tf.nn.convolution semantics: cross-correlation,
    zero 'SAME' padding (extra element at the end) or 'VALID'."""
    require_cuda(x)
    if not batched:
        x = x[None]
    num_dim = x.dim() - 2
    if np.isscalar(axis):
        axis = [axis]
    axes_space = range(num_dim)
    if axis is None:
        axis = axes_space
    assert all(ax in axes_space for ax in axis), 'non-spatial axis passed'

    def conform(v):
        v = np.ravel(1 if v is None else v).tolist()
        return v * len(axis) if len(v) == 1 else v
    strides, dilations = conform(strides), conform(dilations)
    assert len(strides) == len(axis), 'number of strides and axes differ'
    assert len(dilations) == len(axis), 'number of dilations and axes differ'
    if not isinstance(kernels, (tuple, list)):
        kernels = [kernels]
    if len(kernels) == 1:
        kernels = list(kernels) * len(axis)
    assert len(kernels) == len(axis), 'number of kernels and axes differ'
    if padding.upper() not in ('SAME', 'VALID'):
        raise ValueError(f'unknown padding {padding}')

    y = x
    for ax, k, s, d in zip(axis, kernels, strides, dilations):
        s, d = int(s), int(d)
        if s > 1 and d > 1:
            raise ValueError('strides > 1 not supported in conjunction with dilation_rate > 1')
        kdev = torch.as_tensor(k, dtype=torch.float32).reshape(-1)
        if kdev.device != x.device:
            kdev = kdev.to(x.device)           # (a host kernel costs one small synchronous copy per pass)
        kdev = kdev.contiguous()
        K, n = kdev.numel(), y.shape[ax + 1]
        if padding.upper() == 'SAME':
            n_out, pb = _same_padding(n, K, s, d)
        else:
            n_out, pb = max(-(-(n - (K - 1) * d) // s), 0), 0
        y = _ConvAxisFn.apply(y, kdev, ax + 1, s, d, pb, n_out)
    return y if batched else y[0]


def subsample_indices(width, thick, upsample=True):
    """gather indices of subsample_axis for a drawn thickness (utils.py:812-823), fp32 like TF."""
    f32 = np.float32
    num_slice = int(f32(width) / f32(thick) + f32(0.5))

    def lin(stop, num):
        if num == 1:
            return np.array([0], f32)
        delta = f32(stop) / f32(num - 1)
        out = delta * np.arange(num, dtype=f32)
        out[-1] = f32(stop)
        return out
    ind = (lin(width - 1, num_slice) + f32(0.5)).astype(np.int32)
    if not upsample:
        return ind
    return ind[(lin(num_slice - 1, width) + f32(0.5)).astype(np.int32)]


def gather_axis(x, index, axis):
    """tf.gather(x, index, axis=axis) on the device (nrt_gather_axis_f32)."""
    require_cuda(x)
    x32 = _as_f32(x).contiguous()
    idx = torch.as_tensor(np.asarray(index, dtype=np.int32), device=x.device)
    shp = list(x32.shape)
    outer = int(np.prod(shp[:axis], dtype=np.int64))
    inner = int(np.prod(shp[axis + 1:], dtype=np.int64))
    out = torch.empty(shp[:axis] + [idx.numel()] + shp[axis + 1:], dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib.nrt_gather_axis_f32(ptr(x32), ptr(idx), ptr(out), outer, shp[axis], inner, idx.numel(),
                                      stream_ptr(x.device)))
    return out.to(x.dtype) if x.dtype != torch.float32 else out


def subsample_axis(x, stride_min=1, stride_max=8, axes=None, prob=1, upsample=True, seed=None):
    """Symmetrically subsample along one (randomly drawn) axis with nearest neighbours and
    optionally upsample again (utils.py:754-826).  The axis, the thickness and the Bernoulli
    draw come from a numpy generator seeded with `seed` (TF's random stream cannot be
    reproduced outside TF); everything downstream of the draws follows the reference."""
    require_cuda(x)
    rand = np.random.default_rng(seed)
    num_dim = x.dim()
    if axes is None:
        axes = range(num_dim)
    if np.isscalar(axes):
        axes = [axes]
    assert all(i in range(num_dim) for i in axes), 'invalid axis passed'
    assert 0 < stride_min and stride_min <= stride_max, 'invalid strides'
    ax = list(axes)[int(rand.integers(0, len(axes)))]
    thick = np.float32(rand.uniform(stride_min, stride_max))
    assert 0 <= prob <= 1, f'{prob} not a probability'
    if prob < 1 and not (rand.uniform() < prob):
        thick = np.float32(1)
    return gather_axis(x, subsample_indices(x.shape[ax], thick, upsample), ax)


def _norm_gamma(x2d, C, mnmx, gamma_u=None, gamma=0.0):
    """[items, n] -> div_no_nan(x - mn, mx - mn) per row (mnmx may be None: no normalisation), then
    pow(., u * (2 gamma) + (1 - gamma)) with gamma_u [items, C] when given (nrt_norm_gamma_f32)."""
    items, n = x2d.shape
    out = torch.empty_like(x2d)
    f32 = np.float32
    with torch.cuda.device(x2d.device):
        check(lib.nrt_norm_gamma_f32(ptr(x2d), int(items), int(n), int(C), ptr(mnmx), ptr(gamma_u),
                                     float(f32(1 - gamma)), float(f32(1 + gamma)), ptr(out), stream_ptr(x2d.device)))
    return out


def minmax_norm(x, axis=None):
    """Min-max normalize x with a safe division (utils.py:953-968): (x - min) / (max - min), 0 where max == min,
    the extrema taken over `axis` (None: all).  Built for axis=None and any set of trailing axes; the extrema
    stay on the device."""
    require_cuda(x)
    if x.requires_grad and torch.is_grad_enabled():
        raise RuntimeError('minmax_norm has no gradient path through the extrema; pass a detached input')
    nd = x.dim()
    if axis is None:
        k = 0
    else:
        axes = sorted({int(a) + nd if int(a) < 0 else int(a) for a in np.ravel(axis)})
        if any(a < 0 or a >= nd for a in axes):
            raise ValueError(f'axis {axis} out of range for a rank-{nd} tensor')
        k = nd - len(axes)
        if axes != list(range(k, nd)):
            raise NotImplementedError(f'minmax_norm: only axis=None or trailing axes are built, got {axis}')
    x32 = _as_f32(x).contiguous()
    items = int(np.prod(x32.shape[:k], dtype=np.int64))
    n = int(np.prod(x32.shape[k:], dtype=np.int64))
    if x32.numel() == 0:
        return x32.clone()
    x2d = x32.reshape(items, n)
    out = _norm_gamma(x2d, 1, _item_stats(x2d, _lib.NRT_STAT_MINMAX)).reshape(x32.shape)
    return out.to(x.dtype) if x.dtype.is_floating_point and x.dtype != torch.float32 else out


from . import augment  # noqa: E402,F401  (ne.utils.augment.*, as in the reference)
