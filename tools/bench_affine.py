#!/usr/bin/env python
"""
tools/bench_affine.py -- time the generator's label warp (nrt_warp_labels_affine_f32) on a 1x160x192x224 label map
with 16 labels and a SynthMorph-like random affine, and print one JSON line.

    python tools/bench_affine.py [--iters 50] [--warmup 5]

The deformation is VecInt(5) and RescaleTransform(2) of an 80x96x112x3 field.  Records:
  (a) the fused kernel with the deformation: 12 B of deformation read, 4 B of label gather, 4 B of store per voxel
  (b) the fused kernel without it: 4 B gather + 4 B store
  (c) the three-stage chain it replaces on the same inputs (dense shift in the fixed op order as torch element-wise
      ops, ComposeTransform, nearest SpatialTransformer), its output compared bit for bit with (a) in the same run;
      and the last two stages alone, the cost when the dense shift is cached (identity affine)
  (d) a full labels_to_image_new call at the defaults, and with aff_shift=30, aff_rotate=45, aff_scale=0.1,
      aff_shear=0.1, axes_flip=True
Bytes are the algorithmic bytes above; the fraction is of the 3.35 TB/s HBM roofline (H100 SXM data sheet, 700 W
card).  Times are CUDA events around `iters` calls after `warmup`.  The card name and power limit are read in the
same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_BPS = 3.35e12
SHAPE = (160, 192, 224)
BOUNDS = dict(aff_shift=30, aff_rotate=45, aff_scale=0.1, aff_shear=0.1, axes_flip=True, vxm_affine=True)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def rec(name, ms, nbytes=None):
    r = {'name': name, 'ms': round(ms, 4)}
    if nbytes is not None:
        t = nbytes / HBM_BPS * 1e3
        r.update(bytes=int(nbytes), roofline_ms=round(t, 4), frac_of_roofline=round(t / ms, 3))
    return r


def dense_shift(mats, shape):
    """The fixed op order of the kernel's shift, as torch element-wise ops (one rounding each)."""
    B, N = mats.shape[:2]
    grid = torch.meshgrid(*[torch.arange(s, dtype=torch.float32, device=mats.device) for s in shape], indexing='ij')
    col = lambda i, k: mats[:, i, k].reshape(B, *[1] * N)          # noqa: E731
    out = []
    for i in range(N):
        s = col(i, 0) * grid[0]
        for k in range(1, N):
            s = s + col(i, k) * grid[k]
        out.append((s + col(i, N)) - grid[i])
    return torch.stack(out, -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_affine needs a CUDA device')
    import neurite_b200 as ne
    from neurite_b200._lib import lib, check, ptr, stream_ptr, i32_array
    dev = torch.device('cuda:0')
    info = card()
    it, wu = args.iters, args.warmup
    V = int(np.prod(SHAPE))
    rng = np.random.default_rng(0)
    x = torch.as_tensor(rng.integers(0, 16, (1, *SHAPE, 1)).astype(np.float32), device=dev)
    vel = torch.as_tensor(rng.uniform(-2, 2, (1, *[s // 2 for s in SHAPE], 3)).astype(np.float32), device=dev)
    d = ne.layers.RescaleTransform(zoom_factor=2)(ne.layers.VecInt(int_steps=5)(vel)).contiguous()
    gen = ne.models.labels_to_image_new(range(16), in_shape=SHAPE, seeds={'mean': 0, 'warp': 1, 'bias': 2}, **BOUNDS)
    plan = gen._draw(x)
    mats = plan['trans'].contiguous()
    out = torch.empty(1, *SHAPE, 1, device=dev)
    st, shp = stream_ptr(dev), i32_array(SHAPE)

    def fused(dd):
        check(lib.nrt_warp_labels_affine_f32(ptr(x), ptr(mats), ptr(dd), ptr(out), 1, 3, shp, shp, st))
        return out

    st_layer = ne.layers.SpatialTransformer(interp_method='nearest', fill_value=0)
    shift = dense_shift(mats, SHAPE)

    def chain(dd, cached=False):
        t = shift if cached else dense_shift(mats, SHAPE)
        if dd is not None:
            t = ne.layers.ComposeTransform()([t, dd])
        return st_layer([x, t.contiguous()])

    same_d = torch.equal(fused(d).clone(), chain(d))
    same_nod = torch.equal(fused(None).clone(), chain(None))
    records = [
        rec('(a) fused label warp with deformation', timed(lambda: fused(d), it, wu), V * 20),
        rec('(b) fused label warp without deformation', timed(lambda: fused(None), it, wu), V * 8),
        rec('(c) three-stage chain: dense shift, ComposeTransform, nearest SpatialTransformer',
            timed(lambda: chain(d), it, wu)),
        rec('(c) ComposeTransform + nearest SpatialTransformer only (dense shift cached)',
            timed(lambda: chain(d, cached=True), it, wu)),
    ]
    for name, kw in (('defaults', {}), ('SynthMorph-like affine bounds', BOUNDS)):
        g = ne.models.labels_to_image_new(range(16), in_shape=SHAPE, seeds={'mean': 0, 'warp': 1, 'bias': 2}, **kw)
        xi = x.to(torch.int32)
        records.append(rec(f'(d) labels_to_image_new full call, {name}, 16 labels', timed(lambda: g(xi), it // 2 + 1,
                                                                                           wu)))
    print(json.dumps({'card': info, 'iters': it, 'bit_exact_vs_chain': {'with_d': same_d, 'without_d': same_nod},
                      'records': records}), flush=True)
    if not (same_d and same_nod):
        raise SystemExit('the fused kernel and the three-stage chain differ')


if __name__ == '__main__':
    main()
