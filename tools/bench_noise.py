#!/usr/bin/env python
"""
tools/bench_noise.py -- time the synthesis noise layers at labels_to_image_new's defaults (160x192x224, batch 1)
and print one JSON line.

    python tools/bench_noise.py [--iters 20] [--warmup 3]

Each record gives ms per call (CUDA events around `iters` calls after `warmup`), the bytes the call has to move
in HBM (draws written once, each blur pass reads and writes its level, each statistic reads it, the level mean
reads every level and writes the output), the blur's tap FMAs, and which roofline binds: bytes over 3.35 TB/s or
FMAs over 33.5 T FMA/s (67 TFLOP/s FP32), both H100 SXM data-sheet figures for a 700 W card.  The card name and
power limit are read in the same run.
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
HBM_BPS, FMA_PS = 3.35e12, 33.5e12


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


def perlin_model(space, C, L, taps):
    """bytes and tap FMAs of one PerlinNoise item: taps[l] = window of level l (all D axes)."""
    m = int(np.prod(space)) * C
    D = len(space)
    nbytes = L * m * 4 * (1 + 1 + 2 * D + 1 + 1) + m * 4   # draw, stat before, D passes, stat after, mean read; write
    fmas = sum(m * D * k for k in taps)
    return nbytes, fmas


def record(name, ms, nbytes, fmas):
    t_b, t_f = nbytes / HBM_BPS * 1e3, fmas / FMA_PS * 1e3
    bound = 'fma' if t_f > t_b else 'hbm'
    return {'name': name, 'ms': round(ms, 4), 'bytes': int(nbytes), 'tap_fmas': int(fmas), 'bound': bound,
            'roofline_ms': round(max(t_b, t_f), 4), 'frac_of_roofline': round(max(t_b, t_f) / ms, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_noise needs a CUDA device')
    import neurite_b200 as ne
    dev = torch.device('cuda:0')
    info = card()
    win = lambda fwhm: int(np.round(fwhm / 2.355 * 3) * 2 + 1)      # noqa: E731
    out = []

    vel = ne.layers.PerlinNoise(shape=(80, 96, 112, 3), noise_min=0.01, noise_max=2, fwhm_min=[4, 4],
                                fwhm_max=[16, 16], reduce='max', axes=-1, seed=0)
    x1 = torch.zeros(1, 1, 1, 1, 1, device=dev)
    ms = timed(lambda: vel(x1), args.iters, args.warmup)
    out.append(record('velocity PerlinNoise 80x96x112x3, 2 levels, fwhm 4-16, max', ms,
                      *perlin_model((80, 96, 112), 3, 2, [win(16)] * 2)))

    img = torch.rand(1, 160, 192, 224, 1, device=dev)
    bias = ne.layers.PerlinNoise(noise_min=0.01, noise_max=1, fwhm_min=32, fwhm_max=64, seed=0)
    ms = timed(lambda: bias(img), args.iters, args.warmup)
    out.append(record('bias PerlinNoise 160x192x224x1, fwhm 32-64 (165 taps), std', ms,
                      *perlin_model((160, 192, 224), 1, 1, [win(64)])))

    gn = ne.layers.GaussianNoise(0.1, 0.2, seed=0)
    ms = timed(lambda: gn(img), args.iters, args.warmup)
    m = img.numel()
    out.append(record('GaussianNoise(0.1, 0.2) 160x192x224x1', ms, m * 4 * 3, 0))   # max|x| read, x read, out write

    rng = np.random.default_rng(0)

    def torch_bias():
        sd = torch.empty((), device=dev).uniform_(0.01, 1)
        n = torch.randn(1, 160, 192, 224, 1, device=dev) * sd
        ks = [ne.utils.gaussian_kernel(float(rng.uniform(32, 64)) / 2.355, windowsize=win(64), device=dev)
              for _ in range(3)]
        b = ne.utils.separable_conv(n, ks, batched=True)
        return b * (n.std(unbiased=False) / b.std(unbiased=False))
    state = torch.cuda.get_rng_state()
    ms = timed(torch_bias, args.iters, args.warmup)
    torch.cuda.set_rng_state(state)
    out.append(record('torch composition of the bias draw (randn + separable_conv + torch std)', ms,
                      *perlin_model((160, 192, 224), 1, 1, [win(64)])))

    lab = torch.randint(0, 16, (1, 160, 192, 224, 1), device=dev).float()
    vecint = ne.layers.VecInt(int_steps=5)
    resc = ne.layers.RescaleTransform(2)
    warp = ne.layers.SpatialTransformer(interp_method='nearest', fill_value=0)

    def deform():
        v = vel(x1)
        return warp([lab, resc(vecint(v))])
    ms = timed(deform, args.iters, args.warmup)
    out.append({'name': 'deformation draw: PerlinNoise -> VecInt(5) -> RescaleTransform(2) -> nearest '
                        'SpatialTransformer of a 160x192x224 label map', 'ms': round(ms, 4)})

    print(json.dumps({'card': info, 'iters': args.iters, 'records': out}), flush=True)


if __name__ == '__main__':
    main()
