// nrt_mi.cu -- soft-quantised joint histograms and mutual information (SURVEY.md 8f-3).
//
// Reference: neurite/tf/metrics.py:41-336 (MutualInformation.maps / channelwise / volumes /
// volume_seg) and neurite/tf/utils/utils.py:1099-1172 (soft_quantize).  The reference
// materialises two [B,V,nb] soft-quantised tensors (2 x 440 MB for one 160x192x224 volume
// pair at nb = 16) and contracts them with a batched matmul.  Here the quantisation is done in
// registers and the [nb,V] x [V,nb] contraction runs on the tensor cores, so a volume pair is
// read exactly once (8 B per voxel).
//
// Tensor-core path: mma.sync m16n8k8 TF32 with the 3-term split
//     a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi,   a_hi = top 11 bits of a, a_lo = a - a_hi
// (relative error 2^-21 per product, far inside the 1e-5 parity tolerance), accumulators
// flushed into fp32 registers every 128 voxels so tensor-core accumulation rounding cannot
// build up, block partials combined in fp64 in a fixed order (deterministic results).
// The output tile is only nb x nb (16..32), so wgmma's 64-row warpgroup tiles would idle most of
// the array; the warp-level mma shape fits the problem.  With soft quantisation the kernel is
// bound by issue slots / MUFU (32 exponentials per voxel pair), not by HBM; with precomputed
// probability maps (segs) it streams 8*nb bytes per voxel and is HBM-bound.
#include "nrt_common.cuh"

#include <math.h>

namespace nrt {
namespace {

constexpr int kMiThreads = 256;
constexpr int kMiWarps = kMiThreads / 32;
constexpr int kMiMaxBlocks = 592;           // 4 CTAs per SM on up to 148 SMs (sizes the workspace)
constexpr int kMiMaxBins = 64;

struct MiOperand {
  const float* p;          // first voxel of item 0 / channel 0
  int64_t batch_stride;    // floats between items
  int64_t vox_stride;      // floats between voxels
  int nb;                  // bins
  int quant;               // 1: p[v] is an intensity, soft-quantised against centers[nb]
                           // 0: p[v*vox_stride + bin] is a probability / similarity map
  const float* centers;    // device, [nb] (quant only)
};

struct MiArgs {
  MiOperand x, y;
  int64_t nv;              // voxels per item
  float neg_alpha;         // -alpha (utils.py:1166)
  float neg_alpha_log2e;   // -alpha * log2(e): exp(-alpha d^2) = 2^(neg_alpha_log2e * d^2)
  float lo, hi;            // clip (utils.py:1158)
  float* partial;          // [items, nblk, PS]
  int32_t* flag;           // set to 1 if a map value is negative (metrics.py:262-263)
  int nblk;
};

// 2^x, denormal results flushed to zero (weights below 1e-38 do not matter)
__device__ __forceinline__ float ex2_ftz(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// values of one operand for one 8-voxel MMA step: bins g + 8r (r < R) x the lane's two voxels.
// vp points at the lane's first voxel of the step; `left` = voxels from there to the end of the item
// (only read when !FULL).
template <int R, bool Q, bool FULL>
__device__ __forceinline__ void mi_fetch(const float* vp, int vs, int left, int g, const float (&cen)[R],
                                         const bool (&binok)[R], float neg_alpha2, bool clip, float lo, float hi,
                                         float (&val)[R][2], bool& negative) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const bool ok = FULL || k < left;
    const float* p = vp + k * vs;
    if (Q) {
      // utils.py:1157-1171: exp(-alpha * square(clip(x) - c)).  An out-of-range voxel becomes a
      // huge intensity whose weight underflows to exactly 0 for every bin.
      float xv = ok ? ld_stream_f(p) : 3.0e38f;
      if (clip && ok) xv = fminf(fmaxf(xv, lo), hi);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float d = xv - cen[r];
        val[r][k] = ex2_ftz(neg_alpha2 * (d * d));
      }
    } else {
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float t = (ok && binok[r]) ? ld_stream_f(p + g + 8 * r) : 0.0f;
        negative |= (t < 0.0f);
        val[r][k] = t;
      }
    }
  }
}

// a = hi + lo with hi = the top 11 significant bits (a valid TF32 operand); the tensor core drops
// the low 13 bits of lo, leaving a relative error of 2^-22 in the 3-term product
__device__ __forceinline__ void split_tf32(float v, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(v) & 0xffffe000u;
  lo = __float_as_uint(v - __uint_as_float(hi));
}

// One CTA = 8 warps; warp w of block b takes 8*SPC-voxel chunks b*8+w, +nblk*8, ...
// grid = (nblk, channels, items)
template <int MT, int NT, bool QX, bool QY, int SPC, int MINB = 1>
__global__ void __launch_bounds__(kMiThreads, MINB) mi_hist_mma_kernel(const MiArgs a) {
  constexpr int RA = 2 * MT;      // A rows per lane (bins g + 8r)
  constexpr int RB = NT;          // B columns per lane
  constexpr int NBX = 16 * MT, NBY = 8 * NT;
  constexpr int CH = 8 * SPC;
  __shared__ float sh_hist[kMiWarps][NBX * NBY];
  __shared__ float sh_sx[kMiWarps][NBX];
  __shared__ float sh_sy[kMiWarps][NBY];

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int item = blockIdx.z, chan = blockIdx.y;
  const float* xi = a.x.p + (int64_t)item * a.x.batch_stride + (QX ? chan : 0);
  const float* yi = a.y.p + (int64_t)item * a.y.batch_stride + (QY ? chan : 0);

  float cx[RA], cy[RB];
  bool okx[RA], oky[RB];
#pragma unroll
  for (int r = 0; r < RA; ++r) {
    okx[r] = (g + 8 * r) < a.x.nb;
    cx[r] = (QX && okx[r]) ? a.x.centers[g + 8 * r] : INFINITY;      // padded bin: weight exp(-inf) = 0
  }
#pragma unroll
  for (int r = 0; r < RB; ++r) {
    oky[r] = (g + 8 * r) < a.y.nb;
    cy[r] = (QY && oky[r]) ? a.y.centers[g + 8 * r] : INFINITY;
  }

  float tot[MT][NT][4], acc[MT][NT][4], sx[RA], sy[RB];
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int i = 0; i < 4; ++i) tot[m][n][i] = acc[m][n][i] = 0.f;
#pragma unroll
  for (int r = 0; r < RA; ++r) sx[r] = 0.f;
#pragma unroll
  for (int r = 0; r < RB; ++r) sy[r] = 0.f;

  bool negative = false;
  const int64_t nq = (a.nv + CH - 1) / CH;
  const int vsx = (int)a.x.vox_stride, vsy = (int)a.y.vox_stride;
  const bool clip = a.lo > -INFINITY || a.hi < INFINITY;
  int since_flush = 0;

  // one 8-voxel MMA step on the lane's weights: marginal sums, 3xTF32 split, 3 MMAs per output tile
  auto mma_step = [&](const float (&avs)[RA][2], const float (&bvs)[RB][2]) {
    uint32_t ah[MT][4], al[MT][4], bh[NT][2], bl[NT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m) {
      // fragment order: (row g, k t), (row g+8, k t), (row g, k t+4), (row g+8, k t+4)
      const float f[4] = {avs[2 * m][0], avs[2 * m + 1][0], avs[2 * m][1], avs[2 * m + 1][1]};
#pragma unroll
      for (int i = 0; i < 4; ++i) split_tf32(f[i], ah[m][i], al[m][i]);
      sx[2 * m] += f[0] + f[2];
      sx[2 * m + 1] += f[1] + f[3];
    }
#pragma unroll
    for (int n = 0; n < NT; ++n) {
#pragma unroll
      for (int i = 0; i < 2; ++i) split_tf32(bvs[n][i], bh[n][i], bl[n][i]);
      sy[n] += bvs[n][0] + bvs[n][1];
    }
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        mma_tf32(acc[m][n], al[m], bh[n]);
        mma_tf32(acc[m][n], ah[m], bl[n]);
        mma_tf32(acc[m][n], ah[m], bh[n]);
      }
  };
  auto flush_if_due = [&]() {
    since_flush += SPC;
    if (since_flush >= 16) {                         // 128 voxels per tensor-core accumulation run
      since_flush = 0;
#pragma unroll
      for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            tot[m][n][i] += acc[m][n][i];
            acc[m][n][i] = 0.f;
          }
    }
  };

  const int64_t qstride = (int64_t)gridDim.x * kMiWarps;
  if constexpr (QX && QY) {
    // Two intensity images: only 2 + 2 floats per lane and step come from memory.  The raw values
    // of the NEXT chunk are loaded before the current chunk's 32 exponentials and 24 MMAs are
    // issued, so the global-load latency hides behind a full chunk of arithmetic.
    auto load_raw = [&](int64_t q, float (&xo)[SPC][2], float (&yo)[SPC][2]) {
      const int64_t v0 = q * CH + 2 * t;            // the lane's voxel pair of step 0: k = t -> v, k = t + 4 -> v + 1
      const float* xq = xi + v0 * a.x.vox_stride;
      const float* yq = yi + v0 * a.y.vox_stride;
      if ((q + 1) * CH <= a.nv) {                   // warp-uniform: every chunk but the last is full
#pragma unroll
        for (int s = 0; s < SPC; ++s)
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            xo[s][k] = ld_stream_f(xq + (s * 8 + k) * vsx);
            yo[s][k] = ld_stream_f(yq + (s * 8 + k) * vsy);
          }
        if (clip) {
#pragma unroll
          for (int s = 0; s < SPC; ++s)
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              xo[s][k] = fminf(fmaxf(xo[s][k], a.lo), a.hi);
              yo[s][k] = fminf(fmaxf(yo[s][k], a.lo), a.hi);
            }
        }
      } else {
        // an out-of-range voxel becomes a huge intensity whose weight underflows to exactly 0
        const int left0 = (int)(a.nv - v0);         // may be <= 0
#pragma unroll
        for (int s = 0; s < SPC; ++s)
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            const bool ok = s * 8 + k < left0;
            xo[s][k] = ok ? fminf(fmaxf(ld_stream_f(xq + (s * 8 + k) * vsx), a.lo), a.hi) : 3.0e38f;
            yo[s][k] = ok ? fminf(fmaxf(ld_stream_f(yq + (s * 8 + k) * vsy), a.lo), a.hi) : 3.0e38f;
          }
      }
    };
    float xr[SPC][2], yr[SPC][2];
    int64_t q = (int64_t)blockIdx.x * kMiWarps + warp;
    if (q < nq) load_raw(q, xr, yr);
    for (; q < nq; q += qstride) {
      float xn[SPC][2], yn[SPC][2];
      const bool more = q + qstride < nq;
      if (more) load_raw(q + qstride, xn, yn);
#pragma unroll
      for (int s = 0; s < SPC; ++s) {
        float avs[RA][2], bvs[RB][2];
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          // utils.py:1157-1171: exp(-alpha * square(clip(x) - c)); padded bins have c = +inf -> weight 0
#pragma unroll
          for (int r = 0; r < RA; ++r) {
            const float d = xr[s][k] - cx[r];
            avs[r][k] = ex2_ftz(a.neg_alpha_log2e * (d * d));
          }
#pragma unroll
          for (int r = 0; r < RB; ++r) {
            const float d = yr[s][k] - cy[r];
            bvs[r][k] = ex2_ftz(a.neg_alpha_log2e * (d * d));
          }
        }
        mma_step(avs, bvs);
      }
      flush_if_due();
      if (more) {
#pragma unroll
        for (int s = 0; s < SPC; ++s)
#pragma unroll
          for (int k = 0; k < 2; ++k) { xr[s][k] = xn[s][k]; yr[s][k] = yn[s][k]; }
      }
    }
  } else {
    for (int64_t q = (int64_t)blockIdx.x * kMiWarps + warp; q < nq; q += qstride) {
      float av[SPC][RA][2], bv[SPC][RB][2];
      const int64_t v0 = q * CH + 2 * t;
      const float* xq = xi + v0 * a.x.vox_stride;
      const float* yq = yi + v0 * a.y.vox_stride;
      if ((q + 1) * CH <= a.nv) {
#pragma unroll
        for (int s = 0; s < SPC; ++s) {             // all loads of the chunk are issued before any use
          mi_fetch<RA, QX, true>(xq + s * 8 * vsx, vsx, 0, g, cx, okx, a.neg_alpha_log2e, clip, a.lo, a.hi, av[s], negative);
          mi_fetch<RB, QY, true>(yq + s * 8 * vsy, vsy, 0, g, cy, oky, a.neg_alpha_log2e, clip, a.lo, a.hi, bv[s], negative);
        }
      } else {
        const int left0 = (int)(a.nv - v0);
#pragma unroll
        for (int s = 0; s < SPC; ++s) {
          mi_fetch<RA, QX, false>(xq + s * 8 * vsx, vsx, left0 - s * 8, g, cx, okx, a.neg_alpha_log2e, clip, a.lo, a.hi, av[s], negative);
          mi_fetch<RB, QY, false>(yq + s * 8 * vsy, vsy, left0 - s * 8, g, cy, oky, a.neg_alpha_log2e, clip, a.lo, a.hi, bv[s], negative);
        }
      }
#pragma unroll
      for (int s = 0; s < SPC; ++s) mma_step(av[s], bv[s]);
      flush_if_due();
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int i = 0; i < 4; ++i) tot[m][n][i] += acc[m][n][i];

  // marginal sums: the 4 lanes of a group hold different voxels of the same bins
#pragma unroll
  for (int r = 0; r < RA; ++r) {
    sx[r] += __shfl_xor_sync(0xffffffffu, sx[r], 1);
    sx[r] += __shfl_xor_sync(0xffffffffu, sx[r], 2);
  }
#pragma unroll
  for (int r = 0; r < RB; ++r) {
    sy[r] += __shfl_xor_sync(0xffffffffu, sy[r], 1);
    sy[r] += __shfl_xor_sync(0xffffffffu, sy[r], 2);
  }
  // accumulator layout: [0] (g, 2t) [1] (g, 2t+1) [2] (g+8, 2t) [3] (g+8, 2t+1)
#pragma unroll
  for (int m = 0; m < MT; ++m)
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const int i0 = 16 * m + g, j0 = 8 * n + 2 * t;
      sh_hist[warp][i0 * NBY + j0] = tot[m][n][0];
      sh_hist[warp][i0 * NBY + j0 + 1] = tot[m][n][1];
      sh_hist[warp][(i0 + 8) * NBY + j0] = tot[m][n][2];
      sh_hist[warp][(i0 + 8) * NBY + j0 + 1] = tot[m][n][3];
    }
  if (t == 0) {
#pragma unroll
    for (int r = 0; r < RA; ++r) sh_sx[warp][g + 8 * r] = sx[r];
#pragma unroll
    for (int r = 0; r < RB; ++r) sh_sy[warp][g + 8 * r] = sy[r];
  }
  if (negative && a.flag) *a.flag = 1;
  __syncthreads();

  const int nbx = a.x.nb, nby = a.y.nb;
  const int PS = nbx * nby + nbx + nby;
  float* out = a.partial + ((int64_t)(item * gridDim.y + chan) * gridDim.x + blockIdx.x) * PS;
  for (int idx = threadIdx.x; idx < PS; idx += kMiThreads) {
    float s = 0.f;
    if (idx < nbx * nby) {
      const int i = idx / nby, j = idx - i * nby;
#pragma unroll
      for (int w = 0; w < kMiWarps; ++w) s += sh_hist[w][i * NBY + j];
    } else if (idx < nbx * nby + nbx) {
#pragma unroll
      for (int w = 0; w < kMiWarps; ++w) s += sh_sx[w][idx - nbx * nby];
    } else {
#pragma unroll
      for (int w = 0; w < kMiWarps; ++w) s += sh_sy[w][idx - nbx * nby - nbx];
    }
    out[idx] = s;
  }
}

// CUDA-core kernel for any nb <= 64 (and the cross-check of the tensor-core path): 32 voxels
// are soft-quantised into shared memory, then every thread owns (i, j) pairs.
constexpr int kMiGenVox = 32;
__global__ void __launch_bounds__(kMiThreads) mi_hist_generic_kernel(const MiArgs a) {
  __shared__ float xs[kMiGenVox][kMiMaxBins];
  __shared__ float ys[kMiGenVox][kMiMaxBins];
  const int item = blockIdx.z, chan = blockIdx.y;
  const int nbx = a.x.nb, nby = a.y.nb, npair = nbx * nby;
  const float* xi = a.x.p + (int64_t)item * a.x.batch_stride + (a.x.quant ? chan : 0);
  const float* yi = a.y.p + (int64_t)item * a.y.batch_stride + (a.y.quant ? chan : 0);
  constexpr int kPairs = kMiMaxBins * kMiMaxBins / kMiThreads;   // 16
  float acc[kPairs];
#pragma unroll
  for (int k = 0; k < kPairs; ++k) acc[k] = 0.f;
  float msum = 0.f;                                              // threads < nbx: sx ; nbx.. < nbx+nby: sy
  bool negative = false;
  const int64_t nq = (a.nv + kMiGenVox - 1) / kMiGenVox;
  for (int64_t q = blockIdx.x; q < nq; q += gridDim.x) {
    __syncthreads();
    for (int e = threadIdx.x; e < kMiGenVox * (nbx + nby); e += kMiThreads) {
      const bool isx = e < kMiGenVox * nbx;
      const MiOperand& o = isx ? a.x : a.y;
      const int ee = isx ? e : e - kMiGenVox * nbx;
      const int vv = ee / o.nb, bin = ee - vv * o.nb;
      const int64_t v = q * kMiGenVox + vv;
      float val = 0.f;
      if (v < a.nv) {
        const float* vp = (isx ? xi : yi) + v * o.vox_stride;
        if (o.quant) {
          const float d = fminf(fmaxf(vp[0], a.lo), a.hi) - o.centers[bin];
          val = expf(a.neg_alpha * (d * d));
        } else {
          val = vp[bin];
          negative |= (val < 0.f);
        }
      }
      (isx ? xs : ys)[vv][bin] = val;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kPairs; ++k) {
      const int pr = threadIdx.x + k * kMiThreads;
      if (pr < npair) {
        const int i = pr / nby, j = pr - i * nby;
        float s = acc[k];
#pragma unroll 8
        for (int vv = 0; vv < kMiGenVox; ++vv) s = fmaf(xs[vv][i], ys[vv][j], s);
        acc[k] = s;
      }
    }
    if (threadIdx.x < nbx + nby) {
      const bool isx = threadIdx.x < nbx;
      const int bin = isx ? threadIdx.x : threadIdx.x - nbx;
      for (int vv = 0; vv < kMiGenVox; ++vv) msum += (isx ? xs : ys)[vv][bin];
    }
  }
  if (negative && a.flag) *a.flag = 1;
  const int PS = npair + nbx + nby;
  float* out = a.partial + ((int64_t)(item * gridDim.y + chan) * gridDim.x + blockIdx.x) * PS;
#pragma unroll
  for (int k = 0; k < kPairs; ++k) {
    const int pr = threadIdx.x + k * kMiThreads;
    if (pr < npair) out[pr] = acc[k];
  }
  if (threadIdx.x < nbx + nby) out[npair + threadIdx.x] = msum;
}

// stats[item][idx] = sum over blocks (fp64, fixed order).  grid (items, ceil(PS/32)), block (32, 8)
__global__ void mi_combine_kernel(const float* partial, int nblk, int PS, float* stats) {
  __shared__ double sh[8][33];
  const int item = blockIdx.x;
  const int idx = blockIdx.y * 32 + threadIdx.x;
  double s = 0.0;
  if (idx < PS) {
    const float* p = partial + (int64_t)item * nblk * PS + idx;
    for (int b = threadIdx.y; b < nblk; b += 8) s += (double)p[(int64_t)b * PS];
  }
  sh[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && idx < PS) {
    double tot = 0.0;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += sh[w][threadIdx.x];
    stats[(int64_t)item * PS + idx] = (float)tot;
  }
}

__device__ __forceinline__ double block_sum_f64(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < nw; ++w) s += sh[w];
  return s;
}

// metrics.py:265-292 on the raw sums: one block per item.
//   pxy = hist / (sum(hist) + eps) ; px = sx / (sum(sx) + eps) ; py likewise
//   mi  = sum pxy * log(pxy / (px*py + eps) + eps)
__global__ void mi_finalize_kernel(const float* stats, int nbx, int nby, float eps, float* mi) {
  __shared__ double sh[8];
  const int item = blockIdx.x;
  const int npair = nbx * nby, PS = npair + nbx + nby;
  const float* h = stats + (int64_t)item * PS;
  const float* sx = h + npair;
  const float* sy = sx + nbx;
  double th = 0.0, tx = 0.0, ty = 0.0;
  for (int i = threadIdx.x; i < npair; i += blockDim.x) th += (double)h[i];
  for (int i = threadIdx.x; i < nbx; i += blockDim.x) tx += (double)sx[i];
  for (int i = threadIdx.x; i < nby; i += blockDim.x) ty += (double)sy[i];
  const float toth = __fadd_rn((float)block_sum_f64(th, sh), eps);
  const float totx = __fadd_rn((float)block_sum_f64(tx, sh), eps);
  const float toty = __fadd_rn((float)block_sum_f64(ty, sh), eps);
  double acc = 0.0;
  for (int idx = threadIdx.x; idx < npair; idx += blockDim.x) {
    const int i = idx / nby, j = idx - i * nby;
    const float pxy = __fdiv_rn(h[idx], toth);
    const float px = __fdiv_rn(sx[i], totx), py = __fdiv_rn(sy[j], toty);
    const float pxpy_eps = __fadd_rn(__fmul_rn(px, py), eps);
    const float lt = logf(__fadd_rn(__fdiv_rn(pxy, pxpy_eps), eps));
    acc += (double)__fmul_rn(pxy, lt);
  }
  const double tot = block_sum_f64(acc, sh);
  if (threadIdx.x == 0) mi[item] = (float)tot;
}

// tf.linspace(min, max, nb) in fp32: endpoints exact, interior start + delta * i
__global__ void mi_centers_kernel(const float* minmax, int nb, float* centers) {
  const int i = threadIdx.x;
  if (i >= nb) return;
  const float mn = minmax[0], mx = minmax[1];
  if (nb == 1 || i == 0) { centers[i] = mn; return; }
  if (i == nb - 1) { centers[i] = mx; return; }
  const float delta = __fdiv_rn(__fsub_rn(mx, mn), (float)(nb - 1));
  centers[i] = __fadd_rn(mn, __fmul_rn(delta, (float)i));
}

// utils.py:1099-1172 soft_quantize as a tensor op: out[e, b] = exp(-alpha (clip(x[e]) - c[b])^2)
__global__ void soft_quantize_kernel(const float* x, int64_t n, const float* centers, int nb, float neg_alpha, float lo,
                                     float hi, int return_log, float* out) {
  const int64_t total = n * nb;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t v = e / nb;
    const int b = (int)(e - v * nb);
    const float d = __fsub_rn(fminf(fmaxf(x[v], lo), hi), centers[b]);
    const float lg = __fmul_rn(neg_alpha, __fmul_rn(d, d));
    out[e] = return_log ? lg : expf(lg);
  }
}

template <int MT, int NT, int SPC>
void launch_mma(const MiArgs& a, dim3 grid, cudaStream_t st) {
  // two quantised operands: 2 CTAs per SM -- the MUFU and tensor pipes are the limit, more resident warps only add
  // contention
  if (a.x.quant && a.y.quant) mi_hist_mma_kernel<MT, NT, true, true, SPC, 2><<<grid, kMiThreads, 0, st>>>(a);
  else if (a.x.quant) mi_hist_mma_kernel<MT, NT, true, false, SPC><<<grid, kMiThreads, 0, st>>>(a);
  else if (a.y.quant) mi_hist_mma_kernel<MT, NT, false, true, SPC><<<grid, kMiThreads, 0, st>>>(a);
  else mi_hist_mma_kernel<MT, NT, false, false, SPC><<<grid, kMiThreads, 0, st>>>(a);
}

int mi_blocks(int64_t nv, int items) {
  const int per_sm = env_int("NRT_MI_CTAS_PER_SM", 4);
  int64_t want = ((int64_t)sm_count() * (per_sm > 0 ? per_sm : 4) + items - 1) / items;          // ~4 CTAs per SM in total
  int64_t cap = (nv + 1023) / 1024;                                      // >= 1024 voxels per CTA
  int64_t n = want < cap ? want : cap;
  if (n < 1) n = 1;
  if (n > kMiMaxBlocks) n = kMiMaxBlocks;
  return (int)n;
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int64_t nrt_mi_workspace_bytes(int items, int nbx, int nby) {
  if (items < 1 || nbx < 1 || nby < 1) return 0;
  return (int64_t)items * kMiMaxBlocks * ((int64_t)nbx * nby + nbx + nby) * (int64_t)sizeof(float);
}

int nrt_mi_hist_f32(const float* x, int64_t x_batch_stride, int64_t x_vox_stride, int x_quant, int nbx,
                    const float* x_centers, const float* y, int64_t y_batch_stride, int64_t y_vox_stride,
                    int y_quant, int nby, const float* y_centers, int B, int C, int64_t nv, float alpha,
                    float min_clip, float max_clip, float* stats, int32_t* flag, void* workspace,
                    int64_t workspace_bytes, void* stream) {
  NRT_REQUIRE(x && y && stats && workspace, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 1 && C >= 1 && nv >= 0, NRT_E_ARG, "bad B/C/nv");
  NRT_REQUIRE(nbx >= 1 && nby >= 1 && nbx <= kMiMaxBins && nby <= kMiMaxBins, NRT_E_SIZE,
              "bins (%d, %d) outside 1..%d", nbx, nby, kMiMaxBins);
  NRT_REQUIRE(!x_quant || x_centers, NRT_E_ARG, "x_quant needs bin centres");
  NRT_REQUIRE(!y_quant || y_centers, NRT_E_ARG, "y_quant needs bin centres");
  NRT_REQUIRE(C == 1 || (x_quant && y_quant), NRT_E_ARG, "channels > 1 only for two quantised operands");
  NRT_REQUIRE(B <= 65535 && C <= 65535, NRT_E_SIZE, "B or C > 65535");
  NRT_REQUIRE(x_vox_stride >= 1 && y_vox_stride >= 1 && x_vox_stride <= (1 << 20) && y_vox_stride <= (1 << 20),
              NRT_E_SIZE, "voxel strides outside 1..2^20");
  const int items = B * C;
  NRT_REQUIRE(workspace_bytes >= nrt_mi_workspace_bytes(items, nbx, nby), NRT_E_ARG, "workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  MiArgs a;
  a.x = MiOperand{x, x_batch_stride, x_vox_stride, nbx, x_quant, x_centers};
  a.y = MiOperand{y, y_batch_stride, y_vox_stride, nby, y_quant, y_centers};
  a.nv = nv;
  a.neg_alpha = -alpha;
  a.neg_alpha_log2e = (float)(-(double)alpha * 1.4426950408889634);
  a.lo = min_clip;
  a.hi = max_clip;
  a.partial = static_cast<float*>(workspace);
  a.flag = flag;
  const int nblk = mi_blocks(nv, items);
  a.nblk = nblk;
  dim3 grid(nblk, C, B);
  // alpha <= 0 would turn the padded bins' exp(-alpha * inf) into NaN: no padding in the generic kernel
  const bool generic = env_int("NRT_MI_GENERIC", 0) != 0 || nbx > 32 || nby > 32 || !(alpha > 0.f);
  if (generic) {
    mi_hist_generic_kernel<<<grid, kMiThreads, 0, st>>>(a);
  } else if (nbx <= 16 && nby <= 16) {
    launch_mma<1, 2, 4>(a, grid, st);
  } else {
    launch_mma<2, 4, 2>(a, grid, st);                // 32 x 32 bins: 64 accumulators, 2 CTAs per SM
  }
  int rc = check_launch("mi_hist kernel");
  if (rc != NRT_OK) return rc;
  const int PS = nbx * nby + nbx + nby;
  mi_combine_kernel<<<dim3(items, (PS + 31) / 32), dim3(32, 8), 0, st>>>(a.partial, nblk, PS, stats);
  return check_launch("mi_combine_kernel");
}

int nrt_mi_finalize_f32(const float* stats, int items, int nbx, int nby, float eps, float* mi, void* stream) {
  NRT_REQUIRE(stats && mi, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(items >= 1 && nbx >= 1 && nby >= 1, NRT_E_ARG, "bad items/bins");
  mi_finalize_kernel<<<items, 128, 0, static_cast<cudaStream_t>(stream)>>>(stats, nbx, nby, eps, mi);
  return check_launch("mi_finalize_kernel");
}

int nrt_mi_bin_centers_f32(const float* minmax, int nb, float* centers, void* stream) {
  NRT_REQUIRE(minmax && centers, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(nb >= 1 && nb <= 1024, NRT_E_SIZE, "nb = %d outside 1..1024", nb);
  mi_centers_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(minmax, nb, centers);
  return check_launch("mi_centers_kernel");
}

int nrt_soft_quantize_f32(const float* x, int64_t n, const float* centers, int nb, float alpha, float min_clip,
                          float max_clip, int return_log, float* out, void* stream) {
  NRT_REQUIRE(x && centers && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(n >= 0 && nb >= 1, NRT_E_ARG, "bad n/nb");
  if (n == 0) return NRT_OK;
  const int64_t total = n * nb;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 16);
  soft_quantize_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n, centers, nb, -alpha, min_clip, max_clip,
                                                                        return_log, out);
  return check_launch("soft_quantize_kernel");
}

}  // extern "C"
