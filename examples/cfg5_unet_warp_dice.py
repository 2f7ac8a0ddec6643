#!/usr/bin/env python
"""
BASELINE.json configs[4]: UNet forward -> SpatialTransformer -> Dice on synthetic
160x192x224 volumes, one process per GPU.

    python examples/cfg5_unet_warp_dice.py --batch 1
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \
        examples/cfg5_unet_warp_dice.py --batch 8 [--mode slab]

The UNet is context (SURVEY.md 2, row 12): the reference builds it from stock Keras conv /
pool / upsample layers (neurite/tf/models.py:88-246, conv_enc :1309, conv_dec :1445); here
the same topology is written with stock torch (cuDNN) layers only to drive the hot path.
The hot path itself -- the 16-channel warp and the Dice loss -- runs in neurite_b200's CUDA
kernels (z-marching ring kernel, nrt_warp_march.cu; dice_sums kernels, nrt_metrics.cu).

  --mode batch   the global batch is split over the ranks; every rank pushes its own volumes through
                 UNet -> warp -> Dice; the only collective is the all-reduce of the scalar mean loss.
  --mode slab    "8xH100 z-slab shard with halo": EVERY volume of the global batch is split along z over the
                 ranks.  A rank runs the UNet on its slab plus the network's receptive-field margin (24 planes,
                 windows aligned to the pooling stride 8, so the slab's segmentation equals the whole-volume
                 one), keeps only its own planes, exchanges `halo` planes of the 16-channel segmentation with
                 its neighbours while the interior of the slab is warped (neurite_b200.dist.SlabWarper), and
                 all-reduces the [B,16,3] Dice partial sums.

`Cfg5` is importable: bench.py --op cfg5 times the same step (with per-stage CUDA events).
"""
import argparse
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import neurite_b200 as ne  # noqa: E402
from neurite_b200 import dist as nd  # noqa: E402

SHAPE = (160, 192, 224)


class UNet(nn.Module):
    """ne.models.unet topology: nb_levels of [conv3-ELU] + maxpool, mirrored decoder with
    upsample + skip concat, 1x1x1 conv + softmax over nb_labels (models.py:88-246)."""

    def __init__(self, nb_features=16, nb_levels=4, nb_labels=16, feat_mult=2, in_ch=1):
        super().__init__()
        self.enc, self.dec = nn.ModuleList(), nn.ModuleList()
        ch, feats = in_ch, []
        for lvl in range(nb_levels):
            f = int(nb_features * feat_mult ** lvl)
            self.enc.append(nn.Conv3d(ch, f, 3, padding=1))
            feats.append(f)
            ch = f
        for lvl in range(nb_levels - 2, -1, -1):
            f = feats[lvl]
            self.dec.append(nn.Conv3d(ch + f, f, 3, padding=1))
            ch = f
        self.head = nn.Conv3d(ch, nb_labels, 1)
        self.nb_levels = nb_levels

    def forward(self, x):                                   # x [B,1,D,H,W] (channels_last_3d memory)
        skips = []
        for i, conv in enumerate(self.enc):
            x = F.elu(conv(x))
            if i < len(self.enc) - 1:
                skips.append(x)
                x = F.max_pool3d(x, 2)
        for conv in self.dec:
            s = skips.pop()
            x = F.interpolate(x, size=s.shape[2:], mode='nearest')
            x = F.elu(conv(torch.cat([x, s], 1)))
        return torch.softmax(self.head(x), 1)

    def z_margin(self):
        """planes of context a z-window needs on either side so that its interior equals the whole-volume output:
        receptive-field radius of the conv stack (1 + 2 + 4 + ... down, ... + 2 + 1 up), rounded up to the pooling
        stride so that windows can start on a pooling boundary"""
        n = self.nb_levels
        radius = sum(2 ** i for i in range(n)) + sum(2 ** i for i in range(n - 1))
        stride = 2 ** (n - 1)
        return -(-radius // stride) * stride, stride


class Cfg5:
    """One cfg-5 step on this rank.  mode 'batch': `batch` volumes of this rank; mode 'slab': this rank's z-slab of
    every one of `batch` volumes."""

    def __init__(self, mode, batch, dev, world=1, rank=0, group=None, shape=SHAPE, features=16, levels=4, labels=16,
                 flow_amp=3.0, seed=100):
        self.mode, self.B, self.dev, self.world, self.rank, self.group = mode, batch, dev, world, rank, group
        self.S, self.L = tuple(shape), labels
        torch.manual_seed(0)                                  # identical weights on every rank
        self.net = UNet(features, levels, labels).to(dev).to(memory_format=torch.channels_last_3d).eval()
        g = torch.Generator(device=dev).manual_seed(seed + (0 if mode == 'slab' else rank))
        S, B = self.S, batch
        img = torch.randn((B, 1) + S, device=dev, generator=g)
        self.warp = ne.layers.SpatialTransformer()
        self.z0, self.nz = (0, S[0]) if (mode == 'batch' or world == 1) else nd.slab_bounds(S[0], world, rank)
        z0, nz = self.z0, self.nz
        if mode == 'slab' and world > 1:
            margin, stride = self.net.z_margin()
            self.w0 = max(((z0 - margin) // stride) * stride, 0)
            self.w1 = min(-(-(z0 + nz + margin) // stride) * stride, S[0])
            img = img[:, :, self.w0:self.w1]
            # (every rank draws the same global tensors from the same seed and keeps its planes)
            flow = torch.rand((B,) + S + (3,), device=dev, generator=g) * (2 * flow_amp) - flow_amp
            lab = torch.randint(0, labels, (B,) + S, device=dev, generator=g)
            self.flow = flow[:, z0:z0 + nz].contiguous()
            self.target = F.one_hot(lab[:, z0:z0 + nz], labels).float()
            del flow, lab
            self.plan = nd.SlabWarper(S[0], halo=int(flow_amp) + 1 if float(flow_amp).is_integer() else int(flow_amp) + 2,
                                      group=group)
            # (a warped softmax can exceed 1 by an ulp: the reference's range assert is switched off instead of
            #  clamping -- one pass over the tensor and one host sync less per step)
            self.dice = ne.losses.Dice(group=group, check_input_limits=False)
        else:
            self.w0, self.w1 = 0, S[0]
            self.flow = torch.rand((B,) + S + (3,), device=dev, generator=g) * (2 * flow_amp) - flow_amp
            self.target = F.one_hot(torch.randint(0, labels, (B,) + S, device=dev, generator=g), labels).float()
            self.plan = None
            self.dice = ne.losses.Dice(check_input_limits=False)
        self.img = img.contiguous(memory_format=torch.channels_last_3d)
        self.voxels_per_step = B * S[0] * S[1] * S[2] if mode == 'slab' else B * S[0] * S[1] * S[2] * world
        self.events = None

    def unet(self):
        with torch.no_grad(), torch.autocast('cuda', dtype=torch.bfloat16):
            seg = self.net(self.img)                         # [B,L,win,H,W], channels_last_3d memory
        seg = seg[:, :, self.z0 - self.w0:self.z0 - self.w0 + self.nz].permute(0, 2, 3, 4, 1)
        # channels-last view [B,nz,H,W,L]: no transpose, the memory format already is NDHWC; ONE fp32 cast, written
        # straight into the slab plan's source buffer when there is one (no second copy inside the warp step)
        if self.plan is not None:
            dst = self.plan.source_view(torch.empty((seg.shape[0], 0) + tuple(seg.shape[2:]), device=seg.device))
            dst.copy_(seg)
            return dst
        return seg.float().contiguous()

    def step(self, mark=None):
        """returns the scalar mean Dice loss (device tensor).  mark(i) is called after each stage (CUDA events)."""
        seg = self.unet()
        if mark:
            mark(0)
        if self.plan is not None:
            moved = self.plan(seg, self.flow)
        else:
            moved = self.warp([seg, self.flow])
        if mark:
            mark(1)
        loss = self.dice.mean_loss(self.target, moved)
        if self.mode == 'batch' and self.world > 1:
            torch.distributed.all_reduce(loss, group=self.group)
            loss = loss / self.world
        if mark:
            mark(2)
        return loss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=1, help='volumes per rank (batch mode) / per job (slab mode)')
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--features', type=int, default=16)
    ap.add_argument('--levels', type=int, default=4)
    ap.add_argument('--shape', type=int, nargs=3, default=list(SHAPE))
    ap.add_argument('--mode', default='batch', choices=['batch', 'slab'])
    args = ap.parse_args()
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        torch.distributed.init_process_group('nccl', device_id=dev)
    group = torch.distributed.group.WORLD if world > 1 else None
    job = Cfg5(args.mode, args.batch, dev, world, rank, group, tuple(args.shape), args.features, args.levels)
    job.step()
    torch.cuda.synchronize()
    if world > 1:
        torch.distributed.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = job.step()
    e1.record()
    torch.cuda.synchronize()
    if job.plan is not None:
        job.plan.check()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        torch.distributed.all_reduce(ms, op=torch.distributed.ReduceOp.MAX)
    if rank == 0:
        V = args.shape[0] * args.shape[1] * args.shape[2]
        print('cfg5 %s: %d GPU(s), %.1f ms/step, %.2f volumes/s, mean Dice loss %.5f'
              % (args.mode, world, float(ms) / args.steps, job.voxels_per_step / V * args.steps / (float(ms) * 1e-3),
                 float(loss)))
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == '__main__':
    main()
