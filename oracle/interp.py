"""
numpy fp32 restatement of the reference's N-D gridded interpolation.  TEST INFRASTRUCTURE
(see oracle/__init__.py) -- op-for-op, so every intermediate is rounded to fp32 exactly
where TensorFlow would round it (each TF op materialises an fp32 tensor; nothing is fused).

Follows adalca/neurite: neurite/tf/utils/utils.py:
    interpn      :73-220
    resize/zoom  :223-265
    ndgrid/meshgrid/volshape_to_ndgrid/volshape_to_meshgrid  :333-476
    sub2ind2d    :1068-1082
    prod_n       :1085-1092
"""
import itertools

import numpy as np

F32 = np.float32


# ---------------------------------------------------------------------------------------
# helpers (utils.py:1068-1092)
# ---------------------------------------------------------------------------------------
def sub2ind2d(siz, subs):
    """Row-major linearisation, utils.py:1068-1082 (int32 arithmetic like the int32 subs)."""
    assert len(siz) == len(subs), \
        'found inconsistent siz and subs: %d %d' % (len(siz), len(subs))
    k = np.cumprod(siz[::-1])
    ndx = subs[-1]
    for i, v in enumerate(subs[:-1][::-1]):
        ndx = ndx + v * np.int32(k[i])
    return ndx


def prod_n(lst):
    """Chained product ((w0*w1)*w2)..., utils.py:1085-1092.  Not in place (TF tensors are
    immutable, so the reference's `prod *= p` rebinds)."""
    prod = lst[0]
    for p in lst[1:]:
        prod = prod * p
    return prod


# ---------------------------------------------------------------------------------------
# grids (utils.py:333-476)
# ---------------------------------------------------------------------------------------
def meshgrid(*args, indexing='xy'):
    """utils.py:398-476.  Broadcast N rank-1 arrays on an N-D grid ('xy' swaps dims 0/1)."""
    if indexing not in ('xy', 'ij'):
        raise ValueError("indexing parameter must be either 'xy' or 'ij'")
    ndim = len(args)
    s0 = (1,) * ndim
    output = [np.reshape(np.asarray(x), s0[:i] + (-1,) + s0[i + 1:]) for i, x in enumerate(args)]
    sz = [int(np.asarray(x).shape[0]) for x in args]
    if indexing == 'xy' and ndim > 1:
        output[0] = np.reshape(output[0], (1, -1) + (1,) * (ndim - 2))
        output[1] = np.reshape(output[1], (-1, 1) + (1,) * (ndim - 2))
        sz[0], sz[1] = sz[1], sz[0]
    for i in range(len(output)):
        stack_sz = [*sz[:i], 1, *sz[(i + 1):]]
        if indexing == 'xy' and ndim > 1 and i < 2:
            stack_sz[0], stack_sz[1] = stack_sz[1], stack_sz[0]
        output[i] = np.tile(output[i], stack_sz)
    return output


def ndgrid(*args):
    """utils.py:382-395."""
    return meshgrid(*args, indexing='ij')


def volshape_to_ndgrid(volshape):
    """utils.py:333-353."""
    if not all(float(d).is_integer() for d in volshape):
        raise ValueError("volshape needs to be a list of integers")
    return ndgrid(*[np.arange(0, d, dtype=np.int32) for d in volshape])


def volshape_to_meshgrid(volshape, indexing='xy'):
    """utils.py:356-379."""
    if not all(float(d).is_integer() for d in volshape):
        raise ValueError("volshape needs to be a list of integers")
    return meshgrid(*[np.arange(0, d, dtype=np.int32) for d in volshape], indexing=indexing)


def tf_linspace_f32(start, stop, num):
    """tf.linspace in fp32 (third party, TF >= 2.3 math_ops.linspace_nd): endpoints exact,
    interior = start + delta * i with delta = (stop - start) / (num - 1), all in fp32."""
    start, stop = F32(start), F32(stop)
    num = int(num)
    if num == 1:
        return np.array([start], dtype=F32)
    delta = F32(stop - start) / F32(num - 1)
    out = np.empty(num, dtype=F32)
    out[0] = start
    i = np.arange(1, num - 1, dtype=np.int64).astype(F32)
    out[1:num - 1] = start + delta * i
    out[num - 1] = stop
    return out


# ---------------------------------------------------------------------------------------
# interpn (utils.py:73-220)
# ---------------------------------------------------------------------------------------
def interpn(vol, loc, interp_method='linear', fill_value=None):
    """vol: [*S] or [*S, C]; loc: list of D arrays or [*O, D].  Returns [*O] or [*O, C]."""
    if isinstance(loc, (list, tuple)):
        loc = np.stack(loc, -1)                                          # :106-107
    vol = np.asarray(vol)
    loc = np.asarray(loc)
    nb_dims = loc.shape[-1]
    input_vol_shape = vol.shape

    if len(vol.shape) not in [nb_dims, nb_dims + 1]:                     # :111-113
        raise Exception("Number of loc Tensors %d does not match volume dimension %d"
                        % (nb_dims, len(vol.shape[:-1])))
    if nb_dims > len(vol.shape):                                         # :115-117
        raise Exception("Loc dimension %d does not match volume dimension %d"
                        % (nb_dims, len(vol.shape)))
    if len(vol.shape) == nb_dims:                                        # :119-120
        vol = vol[..., None]

    # :123-127 loc takes the volume's float dtype
    vol_is_float = np.issubdtype(vol.dtype, np.floating)
    if not np.issubdtype(loc.dtype, np.floating):
        loc = loc.astype(vol.dtype if vol_is_float else F32)
    elif vol_is_float and vol.dtype != loc.dtype:
        loc = loc.astype(vol.dtype)
    ft = loc.dtype.type

    volshape = list(vol.shape)
    max_loc = [d - 1 for d in volshape]                                  # :134 (channel entry unused)
    vol_reshape = np.reshape(vol, [-1, volshape[-1]])                    # :177

    if interp_method == 'linear':
        loc0 = np.floor(loc)                                             # :139
        clipped_loc = [np.clip(loc[..., d], ft(0), ft(max_loc[d])) for d in range(nb_dims)]     # :142
        loc0lst = [np.clip(loc0[..., d], ft(0), ft(max_loc[d])) for d in range(nb_dims)]        # :143
        loc1 = [np.clip(loc0lst[d] + ft(1), ft(0), ft(max_loc[d])) for d in range(nb_dims)]     # :146
        locs = [[f.astype(np.int32) for f in loc0lst], [f.astype(np.int32) for f in loc1]]      # :147
        diff_loc1 = [loc1[d] - clipped_loc[d] for d in range(nb_dims)]   # :152
        diff_loc0 = [ft(1) - d for d in diff_loc1]                       # :153
        weights_loc = [diff_loc1, diff_loc0]                             # :155

        cube_pts = list(itertools.product([0, 1], repeat=nb_dims))       # :159
        interp_vol = 0                                                   # :160
        for c in cube_pts:                                               # :162
            subs = [locs[c[d]][d] for d in range(nb_dims)]               # :170
            idx = sub2ind2d(vol.shape[:-1], subs)                        # :176
            vol_val = vol_reshape[idx]                                   # :178 tf.gather
            wts_lst = [weights_loc[c[d]][d] for d in range(nb_dims)]     # :183
            wt = prod_n(wts_lst)[..., None]                              # :187-188
            interp_vol = interp_vol + wt * vol_val                       # :191 (mul rounds, then add rounds)
    else:
        assert interp_method == 'nearest', \
            'method should be linear or nearest, got: %s' % interp_method
        # :196 tf.round is half-to-even (np.rint); cast BEFORE clip
        roundloc = np.rint(loc).astype(np.int32)
        roundloc = [np.clip(roundloc[..., d], 0, max_loc[d]) for d in range(nb_dims)]           # :197
        idx = sub2ind2d(vol.shape[:-1], roundloc)                        # :203
        interp_vol = vol_reshape[idx]                                    # :204

    if fill_value is not None:                                           # :206-213
        out_type = interp_vol.dtype.type
        fill_value = out_type(fill_value)
        below = [loc[..., d] < 0 for d in range(nb_dims)]
        above = [loc[..., d] > max_loc[d] for d in range(nb_dims)]
        out_of_bounds = np.any(np.stack(below + above, axis=-1), axis=-1, keepdims=True)
        interp_vol = interp_vol * np.logical_not(out_of_bounds).astype(interp_vol.dtype)
        interp_vol = interp_vol + out_of_bounds.astype(interp_vol.dtype) * fill_value

    if len(input_vol_shape) == nb_dims:                                  # :216-218
        assert interp_vol.shape[-1] == 1, 'Something went wrong with interpn channels'
        interp_vol = interp_vol[..., 0]
    return interp_vol


# ---------------------------------------------------------------------------------------
# resize / zoom (utils.py:223-265)
# ---------------------------------------------------------------------------------------
def resize(vol, zoom_factor, interp_method='linear'):
    vol = np.asarray(vol)
    if isinstance(zoom_factor, (list, tuple)):
        ndims = len(zoom_factor)
        vol_shape = vol.shape[:ndims]
        assert len(vol_shape) in (ndims, ndims + 1), \
            "zoom_factor length %d does not match ndims %d" % (len(vol_shape), ndims)
    else:
        vol_shape = vol.shape[:-1]
        ndims = len(vol_shape)
        zoom_factor = [zoom_factor] * ndims
    if all(z == 1 for z in zoom_factor):                                 # :250-251
        return vol
    new_shape = [int(vol_shape[f] * zoom_factor[f]) for f in range(ndims)]   # :256-257
    lin = [tf_linspace_f32(0., vol_shape[d] - 1., new_shape[d]) for d in range(ndims)]   # :259
    grid = ndgrid(*lin)                                                  # :260
    return interpn(vol, grid, interp_method=interp_method)               # :262


zoom = resize


def resize_layer(x, zoom_factor, interp_method='linear'):
    """layers.Resize.call, layers.py:154-181: per-batch map of resize over [B,*S,C]."""
    x = np.asarray(x)
    ndims = x.ndim - 2
    if not isinstance(zoom_factor, (list, tuple)):
        zoom_factor = [zoom_factor] * ndims
    else:
        assert len(zoom_factor) == ndims, \
            'zoom factor length {} does not match number of dimensions {}'.format(len(zoom_factor), ndims)
    return np.stack([resize(x[b], list(zoom_factor), interp_method) for b in range(x.shape[0])], 0)


# ---------------------------------------------------------------------------------------
# SpatialTransformer (voxelmorph, third party -- contract in SURVEY.md 8c; UNPINNED)
# ---------------------------------------------------------------------------------------
def transform(vol, loc_shift, interp_method='linear', indexing='ij', fill_value=None):
    """vxm.utils.transform: loc = ndgrid(arange(S)) + shift ; interpn.  vol [*S, C], shift [*S, D]."""
    vol = np.asarray(vol)
    loc_shift = np.asarray(loc_shift)
    volshape = loc_shift.shape[:-1]
    nb_dims = len(volshape)
    mesh = volshape_to_meshgrid(volshape, indexing=indexing)
    loc = [mesh[d].astype(loc_shift.dtype) + loc_shift[..., d] for d in range(nb_dims)]
    return interpn(vol, loc, interp_method=interp_method, fill_value=fill_value)


def spatial_transformer(vol, trf, interp_method='linear', indexing='ij', fill_value=None):
    """vxm.layers.SpatialTransformer.call on a dense shift: vol [B,*S,C], trf [B,*S,D].
    'xy' indexing swaps the first two flow channels before use (vxm layers.py)."""
    vol = np.asarray(vol)
    trf = np.asarray(trf)
    if indexing == 'xy':
        trf = np.concatenate([trf[..., 1:2], trf[..., 0:1], trf[..., 2:]], -1)
    return np.stack([transform(vol[b], trf[b], interp_method, 'ij', fill_value)
                     for b in range(vol.shape[0])], 0)


# ---------------------------------------------------------------------------------------
# voxelmorph-adjacent compositions of the warp (SURVEY.md 8f item 2; third party, UNPINNED)
# call sites in the reference: VecInt neurite/tf/models.py:802, 1149; RescaleTransform /
# Resize of the half-resolution field :803-804
# ---------------------------------------------------------------------------------------
def vec_int(vel, int_steps=7, indexing='ij'):
    """vxm.layers.VecInt(method='ss'): scaling and squaring.  vel [B,*S,D] -> displacement."""
    out = []
    for b in range(vel.shape[0]):
        v = (np.asarray(vel[b], dtype=F32) / F32(2 ** int_steps)).astype(F32)
        for _ in range(int_steps):
            v = (v + transform(v, v, 'linear', indexing)).astype(F32)
        out.append(v)
    return np.stack(out, 0)


def compose(transforms, interp_method='linear', indexing='ij'):
    """vxm.utils.compose for dense shifts [*S,D]: T = t_0 o t_1 o ... (right-most applied first)."""
    curr = np.asarray(transforms[-1], dtype=F32)
    for nxt in reversed(transforms[:-1]):
        curr = (curr + transform(np.asarray(nxt, dtype=F32), curr, interp_method, indexing)).astype(F32)
    return curr


def rescale_transform(trf, zoom_factor, interp_method='linear'):
    """vxm.layers.RescaleTransform on dense shifts [B,*S,D]: resize the field and scale its values."""
    z = F32(zoom_factor)
    if zoom_factor < 1:
        return (resize_layer(trf, zoom_factor, interp_method) * z).astype(F32)
    return resize_layer((np.asarray(trf, dtype=F32) * z).astype(F32), zoom_factor, interp_method)
