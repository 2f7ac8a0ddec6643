#!/usr/bin/env python
"""
tools/bench_synth.py -- time labels_to_image_new at its defaults (one-hot on) on a 1x160x192x224 label map with
16 and with 32 labels, and print one JSON line.

    python tools/bench_synth.py [--iters 20] [--warmup 3]

Per label count: ms per full generator call; ms, algorithmic bytes and the fraction of the 3.35 TB/s HBM roofline
(H100 SXM data sheet, 700 W card) for the label-to-image kernel (1), the per-item min/max plus normalise-and-gamma
pair (3) and the one-hot writer (4); and the same stages as a torch composition (gather, exp, amin/amax, pow,
F.one_hot).  Times are CUDA events around `iters` calls after `warmup`.  The card name and power limit are read
in the same run.
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


def rec(name, ms, nbytes):
    t = nbytes / HBM_BPS * 1e3
    return {'name': name, 'ms': round(ms, 4), 'bytes': int(nbytes), 'roofline_ms': round(t, 4),
            'frac_of_roofline': round(t / ms, 3)}


def bench(M, iters, warmup):
    import neurite_b200 as ne
    from neurite_b200._lib import lib, check, ptr, stream_ptr
    dev = torch.device('cuda:0')
    V = int(np.prod(SHAPE))
    gen = ne.models.labels_to_image_new(range(M), in_shape=SHAPE, seeds={'mean': 0, 'warp': 1, 'bias': 2})
    x = torch.randint(0, M, (1, *SHAPE, 1), device=dev, dtype=torch.int32)
    out = [{'name': f'labels_to_image_new defaults, {M} labels, full call', 'ms': round(timed(lambda: gen(x),
                                                                                               iters, warmup), 4)}]
    plan = gen._draw(x)
    warped, _ = gen.warp_labels(x, plan)
    gl, _, mmin, mmax = gen._luts(dev)
    mmin1, mmax1 = mmin[0], mmax[0]
    st = stream_ptr(dev)
    img = torch.empty(1, *SHAPE, 1, device=dev)
    amax = torch.empty(1, device=dev)
    nb = lib.nrt_labels_to_image_workspace_bytes()
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    bias = plan['bias'].contiguous()

    def k1():
        check(lib.nrt_labels_to_image_f32(ptr(warped), 1, V, 1, 1, 1, 0, 1, ptr(gl), gl.numel(), M,
                                          ptr(plan['mean_u']), ptr(mmin), ptr(mmax), ptr(bias), 1, ptr(img), None,
                                          None, ptr(amax), ptr(ws), nb, st))
    out.append(rec('1 labels_to_image (label read, bias read, image write)', timed(k1, iters, warmup), V * 12))

    x2d = img.reshape(1, -1)
    gu = plan['gamma_u']

    def k3():
        mm = ne.utils._item_stats(x2d, ne._lib.NRT_STAT_MINMAX)
        return ne.utils._norm_gamma(x2d, 1, mm, gu, 0.5)
    out.append(rec('3 min/max + normalise + gamma (two reads, one write)', timed(k3, iters, warmup), V * 12))

    oh = torch.empty(1, *SHAPE, M, device=dev)

    def k4():
        check(lib.nrt_label_map_f32(ptr(warped), 1, V, 1, 1, 0, 1, None, 0, M, ptr(oh), st))
    out.append(rec(f'4 one-hot [V, {M}] (label read, 4M bytes written per voxel)', timed(k4, iters, warmup),
                   V * (4 + 4 * M)))

    glong = gl.long()
    mean_u = plan['mean_u'][0, 0]

    def torch_stages():
        idx = glong[warped[..., 0].long()]
        mean = torch.gather(mean_u, 0, idx.reshape(-1)).reshape(idx.shape)[..., None] * (mmax1[idx] - mmin1[idx])[..., None] \
            + mmin1[idx][..., None]
        im = mean * torch.exp(bias)
        mn, mx = im.amin(), im.amax()
        im = ((im - mn) / (mx - mn)).pow(gu[0, 0])
        return im, torch.nn.functional.one_hot(warped[..., 0].long(), M).float()
    out.append({'name': 'torch composition of stages 1, 3, 4 (gather, exp, amin/amax, pow, F.one_hot)',
                'ms': round(timed(torch_stages, iters, warmup), 4)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_synth needs a CUDA device')
    info = card()
    records = bench(16, args.iters, args.warmup) + bench(32, args.iters, args.warmup)
    print(json.dumps({'card': info, 'iters': args.iters, 'records': records}), flush=True)


if __name__ == '__main__':
    main()
