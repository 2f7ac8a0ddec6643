"""
The affine stage of labels_to_image_new.  TEST INFRASTRUCTURE (see oracle/__init__.py).

    params_from_draws       voxelmorph DrawAffineParams on replayed draws (tools/tfshim.py, tools/vxmstub.py): per
                            kind with a non-zero bound, one [B, n] draw; uniform u * (2b) - b, normal z * b, the
                            normal scale redrawn where |z| > 2 (each redraw one more [B, n] draw)
    affine_matrix           ParamsToAffineMatrix(deg=True, shift_scale=True, last_row=True): A = R (Z S)
    flip_matrix, swap_matrix  draw_flip_matrix(shift_center=False) / draw_swap_matrix given their draws
    compose                 models.py:1107-1128: inv(origin) A origin center scale [flip] [swap], fp64
    dense_shift             AffineToDenseShift(shift_center=False) in the fixed order
                            s_i(c) = ((M_i0 c_0 + M_i1 c_1) + M_i2 c_2) + M_iN - c_i, fp32, one rounding per op
    warp_labels             the generator's label warp: ComposeTransform([dense_shift, d]) when there is a
                            deformation, then the nearest SpatialTransformer with fill 0 (oracle/interp.py)

Provenance: contract.  voxelmorph is not part of the reference; these restate its public definitions as the
project fixes them (DESIGN.md §2).  The tests/golden/affsynth_* fixtures run the reference's own
labels_to_image_new with tools/vxmstub.py as voxelmorph, which calls these functions.
"""
import numpy as np

from . import interp as ointerp, synth as osynth

F32 = np.float32
KINDS = (('shift', 'aff_shift', 'aff_normal_shift'), ('rot', 'aff_rotate', 'aff_normal_rotate'),
         ('scale', 'aff_scale', 'aff_normal_scale'), ('shear', 'aff_shear', 'aff_normal_shear'))
AFF_KEYS = tuple(k for _, b, n in KINDS for k in (b, n)) + ('axes_flip', 'axes_swap')


def sizes(ndims):
    r = 3 if ndims == 3 else 1
    return {'shift': ndims, 'rot': r, 'scale': ndims, 'shear': r}


def params_from_draws(q, k, kwargs, batch, ndims):
    """-> ([batch, 12 | 6] fp32 parameters, next draw index)."""
    out = []
    for kind, bkey, nkey in KINDS:
        b, n = kwargs.get(bkey, 0), sizes(ndims)[kind]
        if b == 0:
            out.append(np.zeros((batch, n), F32))
            continue
        if not kwargs.get(nkey, False):
            lo, hi = F32(-b), F32(b)
            out.append((np.asarray(q[k], F32) * F32(hi - lo) + lo).astype(F32))
            k += 1
            continue
        z = np.asarray(q[k], F32).copy()
        k += 1
        while kind == 'scale' and np.any(np.abs(z) > 2):
            z = np.where(np.abs(z) > 2, np.asarray(q[k], F32), z)
            k += 1
        out.append((z * F32(b) + F32(0)).astype(F32))
    return np.concatenate(out, 1), k


def _rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    m = np.eye(3)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    m[i, i], m[j, j] = c, c
    m[i, j], m[j, i] = (-s, s) if axis != 1 else (s, -s)
    return m


def affine_matrix(params, ndims):
    """[B, N+1, N+1] fp32, evaluated in fp64 and rounded once."""
    p = np.asarray(params, np.float64)
    n = sizes(ndims)
    out = np.zeros((p.shape[0], ndims + 1, ndims + 1))
    for b, row in enumerate(p):
        shift = row[:ndims]
        deg = row[ndims:ndims + n['rot']]
        scale = row[ndims + n['rot']:2 * ndims + n['rot']]
        shear = row[2 * ndims + n['rot']:]
        rad = deg * np.pi / 180
        if ndims == 3:
            r = _rot(0, rad[0]) @ (_rot(1, rad[1]) @ _rot(2, rad[2]))
            s = np.eye(3)
            s[0, 1], s[0, 2], s[1, 2] = shear
        else:
            r = _rot(2, rad[0])[:2, :2]
            s = np.eye(2)
            s[0, 1] = shear[0]
        out[b, :ndims, :ndims] = r @ (np.diag(1 + scale) @ s)
        out[b, :ndims, ndims] = shift
        out[b, ndims, ndims] = 1
    return out.astype(F32)


def flip_matrix(u, out_shape):
    """draw_flip_matrix(out_shape, shift_center=False) from its U[0, 1) draw [N]: axis i flips where u_i > 0.5."""
    n = len(out_shape)
    m = np.eye(n + 1)
    for i in range(n):
        if np.asarray(u, F32)[i] > F32(0.5):
            m[i, i], m[i, n] = -1, out_shape[i] - 1
    return m


def swap_matrix(u):
    """draw_swap_matrix from its U[0, 1) draw [N]: perm = the stable argsort of the draw, P[i, perm[i]] = 1."""
    perm = np.argsort(np.asarray(u, F32), kind='stable')
    n = len(perm)
    m = np.eye(n + 1)
    m[:n, :n] = np.eye(n)[perm]
    return m


def compose(aff, in_shape, out_shape, half_res, flip=None, swap=None):
    """[B, N+1, N+1] fp64 (no rounding): inv(origin) @ A @ origin @ center @ scale [@ flip] [@ swap]."""
    in_shape, out_shape = np.asarray(in_shape), np.asarray(out_shape)
    n = len(in_shape)
    origin = np.eye(n + 1)
    origin[:n, -1] = -0.5 * (in_shape - 1)
    center = np.eye(n + 1)
    center[:n, -1] = np.round(0.5 * (in_shape - (2 if half_res else 1) * out_shape))
    scale = np.diag((*[2 if half_res else 1] * n, 1))
    m = np.linalg.inv(origin) @ np.asarray(aff, np.float64) @ origin @ center @ scale
    for f in (flip, swap):
        if f is not None:
            m = m @ f
    return m


def dense_shift(mat, out_shape):
    """mat [N, N+1] fp32 -> the dense shift [*out_shape, N] fp32 in the fixed op order."""
    mat = np.asarray(mat, F32)
    n = len(out_shape)
    grid = np.meshgrid(*[np.arange(s, dtype=F32) for s in out_shape], indexing='ij')
    out = []
    for i in range(n):
        s = (mat[i, 0] * grid[0]).astype(F32)
        for k in range(1, n):
            s = (s + (mat[i, k] * grid[k]).astype(F32)).astype(F32)
        out.append(((s + mat[i, n]).astype(F32) - grid[i]).astype(F32))
    return np.stack(out, -1)


def warp_labels(labels, mats, d, out_shape):
    """labels [B, *in_shape, 1], mats [B, N, N+1], d [B, *out_shape, N] or None -> [B, *out_shape, 1] fp32."""
    out_shape = [int(s) for s in out_shape]
    trf = np.stack([dense_shift(m, out_shape) for m in mats], 0)
    if d is not None:
        trf = np.stack([ointerp.compose([trf[b], np.asarray(d[b], F32)]) for b in range(trf.shape[0])], 0)
    return ointerp.spatial_transformer(np.asarray(labels, F32), trf, 'nearest', fill_value=0).astype(F32)


# ---------------------------------------------------------------------------------------
# the generator with the affine given its draws (tests/golden/affsynth_*)
# ---------------------------------------------------------------------------------------
def decode(kwargs, labels, q):
    """An affsynth_* fixture's arguments, labels and draws -> (cfg, plan, affine) with affine = dict(params, aff
    [B, N+1, N+1] fp32, flip, swap (fp64 matrices or None)); cfg and plan as oracle.synth.decode_synth."""
    B, N = labels.shape[0], len(kwargs['in_shape'])
    params, k = params_from_draws(q, 0, kwargs, B, N)
    c = dict(osynth.SYNTH_DEFAULTS, **{key: v for key, v in kwargs.items() if key not in AFF_KEYS})
    half = c['half_res']
    in_shape = np.asarray(kwargs['in_shape'])
    out_shape = np.array(in_shape if c['out_shape'] is None else c['out_shape']) // (2 if half else 1)
    flip = swap = None
    if kwargs.get('axes_flip'):
        flip, k = flip_matrix(q[k], out_shape), k + 1
    if kwargs.get('axes_swap'):
        swap, k = swap_matrix(q[k]), k + 1
    c, p = osynth.decode_synth({key: v for key, v in kwargs.items() if key not in AFF_KEYS}, labels, q[k:])
    aff = dict(params=params, aff=affine_matrix(params, N), flip=flip, swap=swap)
    return c, p, aff


def synth(labels, c, p, mats, z=None):
    """oracle.synth.synth_from_plan with the affine label warp: the stages after the warp are the same code, run
    on the warped map with an identity geometry."""
    d = None
    if p['vel'] is not None:
        d = ointerp.vec_int(p['vel'], int_steps=5)
        if not c['half_res']:
            d = ointerp.rescale_transform(d, 2)
    warped = warp_labels(labels, mats, d, c['out_shape_eff'])
    ident = dict(c, in_shape=list(c['out_shape_eff']), half_res=False)
    r = osynth.synth_from_plan(warped, ident, dict(p, vel=None), z=z)
    assert np.array_equal(r['warped'], warped)
    if d is not None:
        r['def'] = d
    return r


def outputs(kwargs, r, p, aff):
    """The reference's outputs in its order (models.py:1284-1298)."""
    c = dict(return_im=True, return_map=True, return_vel=False, return_def=False, return_aff=False,
             return_mean=False, return_bias=False)
    c.update(kwargs)
    out = []
    for key, v in (('return_im', r['image']), ('return_map', r['map']), ('return_vel', p['vel']),
                   ('return_def', r.get('def')), ('return_aff', aff), ('return_mean', r['mean']),
                   ('return_bias', r.get('bias'))):
        if c[key]:
            out.append(v)
    return out
