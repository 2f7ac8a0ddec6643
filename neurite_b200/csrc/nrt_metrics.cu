// nrt_metrics.cu -- Dice partial sums / finalize, hard-Dice label counts, argmax, and the
// label-weighted categorical cross-entropy, for sm_90a.
//
// All of these are pure HBM streams (8 B per (voxel,label), SURVEY.md 8d): coalesced
// 128-bit loads that bypass L1, several independent loads in flight per thread, fixed
// label slot per thread so the per-label sums stay in registers, a deterministic two-level
// reduction (block partials in the caller's workspace, fp64 combine) -- no atomics on data.
#include "nrt_common.cuh"

namespace nrt {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 2048;          // per batch item, bounds the workspace

// ---------------------------------------------------------------------------------------
// Dice sums, vector path: L % 4 == 0, q = L/4 divides the active thread count
// ---------------------------------------------------------------------------------------
template <int UNROLL>
__global__ void __launch_bounds__(kThreads)
dice_sums_vec4_kernel(const float4* __restrict__ t4, const float4* __restrict__ p4, int64_t row4,
                      int64_t begin4, int64_t n4, int q, int nthr, int check,
                      float* __restrict__ partial, int32_t* __restrict__ flag) {
  // grid: (blocks, B).  Block `bx` owns float4s [begin4 + bx*per, ...) of batch row `b`.
  __shared__ float s_acc[kThreads][13];
  const int b = blockIdx.y;
  const int tid = threadIdx.x;
  const int64_t per = ((n4 + gridDim.x - 1) / gridDim.x + (int64_t)nthr * UNROLL - 1) /
                      ((int64_t)nthr * UNROLL) * ((int64_t)nthr * UNROLL);
  const int64_t lo = (int64_t)blockIdx.x * per;
  const int64_t hi = min(lo + per, n4);
  const float4* tb = t4 + (int64_t)b * row4 + begin4;
  const float4* pb = p4 + (int64_t)b * row4 + begin4;
  float tp[4] = {0, 0, 0, 0}, tt[4] = {0, 0, 0, 0}, pp[4] = {0, 0, 0, 0};
  bool bad = false;
  if (tid < nthr) {
    int64_t i = lo + tid;
    for (; i + (int64_t)(UNROLL - 1) * nthr < hi; i += (int64_t)UNROLL * nthr) {
      float4 a[UNROLL], c[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) { a[u] = ld_stream_f4(tb + i + (int64_t)u * nthr); c[u] = ld_stream_f4(pb + i + (int64_t)u * nthr); }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        tp[0] += a[u].x * c[u].x; tp[1] += a[u].y * c[u].y; tp[2] += a[u].z * c[u].z; tp[3] += a[u].w * c[u].w;
        tt[0] += a[u].x * a[u].x; tt[1] += a[u].y * a[u].y; tt[2] += a[u].z * a[u].z; tt[3] += a[u].w * a[u].w;
        pp[0] += c[u].x * c[u].x; pp[1] += c[u].y * c[u].y; pp[2] += c[u].z * c[u].z; pp[3] += c[u].w * c[u].w;
        if (check) {
          bad |= !(a[u].x >= 0.f && a[u].x <= 1.f) | !(a[u].y >= 0.f && a[u].y <= 1.f) | !(a[u].z >= 0.f && a[u].z <= 1.f) | !(a[u].w >= 0.f && a[u].w <= 1.f);
          bad |= !(c[u].x >= 0.f && c[u].x <= 1.f) | !(c[u].y >= 0.f && c[u].y <= 1.f) | !(c[u].z >= 0.f && c[u].z <= 1.f) | !(c[u].w >= 0.f && c[u].w <= 1.f);
        }
      }
    }
    for (; i < hi; i += nthr) {
      const float4 a = ld_stream_f4(tb + i), c = ld_stream_f4(pb + i);
      tp[0] += a.x * c.x; tp[1] += a.y * c.y; tp[2] += a.z * c.z; tp[3] += a.w * c.w;
      tt[0] += a.x * a.x; tt[1] += a.y * a.y; tt[2] += a.z * a.z; tt[3] += a.w * a.w;
      pp[0] += c.x * c.x; pp[1] += c.y * c.y; pp[2] += c.z * c.z; pp[3] += c.w * c.w;
      if (check) {
        bad |= !(a.x >= 0.f && a.x <= 1.f) | !(a.y >= 0.f && a.y <= 1.f) | !(a.z >= 0.f && a.z <= 1.f) | !(a.w >= 0.f && a.w <= 1.f);
        bad |= !(c.x >= 0.f && c.x <= 1.f) | !(c.y >= 0.f && c.y <= 1.f) | !(c.z >= 0.f && c.z <= 1.f) | !(c.w >= 0.f && c.w <= 1.f);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) { s_acc[tid][k] = tp[k]; s_acc[tid][4 + k] = tt[k]; s_acc[tid][8 + k] = pp[k]; }
  if (bad) atomicOr(flag, 1);
  __syncthreads();
  // thread (kind, label) sums the nthr/q threads that own that label's quad, fixed order
  const int L = 4 * q;
  for (int o = tid; o < 3 * L; o += kThreads) {
    const int kind = o / L, l = o - kind * L;
    const int quad = l >> 2, e = l & 3;
    float s = 0.f;
    for (int j = quad; j < nthr; j += q) s += s_acc[j][kind * 4 + e];
    partial[((int64_t)b * gridDim.x + blockIdx.x) * 3 * L + o] = s;   // [b][blk][kind][l]
  }
}

// scalar path: any L <= kThreads, fixed label per thread
__global__ void __launch_bounds__(kThreads)
dice_sums_scalar_kernel(const float* __restrict__ t, const float* __restrict__ p, int64_t row,
                        int64_t begin, int64_t n, int L, int nthr, int check,
                        float* __restrict__ partial, int32_t* __restrict__ flag) {
  __shared__ float s_acc[kThreads][3];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int64_t per = ((n + gridDim.x - 1) / gridDim.x + nthr - 1) / nthr * nthr;
  const int64_t lo = (int64_t)blockIdx.x * per, hi = min(lo + per, n);
  const float* tb = t + (int64_t)b * row + begin;
  const float* pb = p + (int64_t)b * row + begin;
  float tp = 0, tt = 0, pp = 0;
  bool bad = false;
  if (tid < nthr) {
    for (int64_t i = lo + tid; i < hi; i += nthr) {
      const float a = ld_stream_f(tb + i), c = ld_stream_f(pb + i);
      tp += a * c; tt += a * a; pp += c * c;
      if (check) bad |= !(a >= 0.f && a <= 1.f) | !(c >= 0.f && c <= 1.f);
    }
  }
  s_acc[tid][0] = tp; s_acc[tid][1] = tt; s_acc[tid][2] = pp;
  if (bad) atomicOr(flag, 1);
  __syncthreads();
  for (int o = tid; o < 3 * L; o += kThreads) {
    const int kind = o / L, l = o - kind * L;
    float s = 0.f;
    for (int j = l; j < nthr; j += L) s += s_acc[j][kind];
    partial[((int64_t)b * gridDim.x + blockIdx.x) * 3 * L + o] = s;
  }
}

// per-voxel path: any L, optional renormalisation (metrics.py:434-436); one warp per voxel
__global__ void __launch_bounds__(kThreads)
dice_sums_voxel_kernel(const float* __restrict__ t, const float* __restrict__ p, int64_t V,
                       int64_t v0, int64_t nv, int L, int normalize, int check,
                       float* __restrict__ partial, int32_t* __restrict__ flag) {
  extern __shared__ float s_lab[];                    // [3][L] block accumulators
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int o = tid; o < 3 * L; o += kThreads) s_lab[o] = 0.f;
  __syncthreads();
  const int64_t per = (nv + gridDim.x - 1) / gridDim.x;
  const int64_t lo = v0 + (int64_t)blockIdx.x * per, hi = min(lo + per, v0 + nv);
  bool bad = false;
  // each warp walks its voxels; lanes stride the labels; per-label register sums are not
  // possible for arbitrary L, so accumulate into shared memory (one owner lane per label
  // per warp -> the 8 warps collide only through atomicAdd on shared floats).
  for (int64_t v = lo + wid; v < hi; v += kThreads / 32) {
    const float* tr = t + ((int64_t)b * V + v) * L;
    const float* pr = p + ((int64_t)b * V + v) * L;
    float st = 1.f, sp = 1.f;
    if (normalize) {
      float a = 0.f, c = 0.f;
      for (int l = lane; l < L; l += 32) { a += tr[l]; c += pr[l]; }
      st = warp_sum(a); sp = warp_sum(c);
    }
    for (int l = lane; l < L; l += 32) {
      float a = tr[l], c = pr[l];
      if (normalize) { a = (st != 0.f) ? __fdiv_rn(a, st) : 0.f; c = (sp != 0.f) ? __fdiv_rn(c, sp) : 0.f; }
      if (check) bad |= !(a >= 0.f && a <= 1.f) | !(c >= 0.f && c <= 1.f);
      atomicAdd(&s_lab[l], a * c);
      atomicAdd(&s_lab[L + l], a * a);
      atomicAdd(&s_lab[2 * L + l], c * c);
    }
  }
  if (bad) atomicOr(flag, 1);
  __syncthreads();
  for (int o = tid; o < 3 * L; o += kThreads)
    partial[((int64_t)b * gridDim.x + blockIdx.x) * 3 * L + o] = s_lab[o];
}

// hard Dice: integer label maps -> exact counts (metrics.py:450-468 without the one-hot)
__global__ void __launch_bounds__(kThreads)
dice_label_counts_kernel(const int32_t* __restrict__ t, const int32_t* __restrict__ p, int64_t V,
                         int64_t v0, int64_t nv, int L, float* __restrict__ partial) {
  extern __shared__ int s_cnt[];                      // [3][L]
  const int b = blockIdx.y, tid = threadIdx.x;
  for (int o = tid; o < 3 * L; o += kThreads) s_cnt[o] = 0;
  __syncthreads();
  const int64_t per = ((nv + gridDim.x - 1) / gridDim.x + kThreads - 1) / kThreads * kThreads;
  const int64_t lo = v0 + (int64_t)blockIdx.x * per, hi = min(lo + per, v0 + nv);
  const int32_t* tb = t + (int64_t)b * V;
  const int32_t* pb = p + (int64_t)b * V;
  for (int64_t v = lo + tid; v < hi; v += kThreads) {
    const int a = __ldg(tb + v), c = __ldg(pb + v);
    const bool ta = (a >= 0) & (a < L), pc = (c >= 0) & (c < L);
    if (ta) atomicAdd(&s_cnt[L + a], 1);
    if (pc) atomicAdd(&s_cnt[2 * L + c], 1);
    if (ta & (a == c)) atomicAdd(&s_cnt[a], 1);
  }
  __syncthreads();
  for (int o = tid; o < 3 * L; o += kThreads)
    partial[((int64_t)b * gridDim.x + blockIdx.x) * 3 * L + o] = (float)s_cnt[o];
}

// combine block partials [b][blk][kind][l] -> sums [b][l][kind], fp64, fixed order
__global__ void dice_combine_serial_kernel(const float* __restrict__ partial, int nblk, int L,
                                           float* __restrict__ sums) {
  const int b = blockIdx.x;
  for (int o = threadIdx.x; o < 3 * L; o += blockDim.x) {
    double s = 0.0;
    for (int k = 0; k < nblk; ++k) s += (double)partial[((int64_t)b * nblk + k) * 3 * L + o];
    const int kind = o / L, l = o - kind * L;
    sums[((int64_t)b * L + l) * 3 + kind] = (float)s;
  }
}

// The same in two levels (3L <= blockDim): the serial kernel's 48 threads each walk all ~300 block partials, a long
// serial tail behind the streaming kernel.  Here slice s of blockDim / 3L slices sums
// blocks s, s + nslice, ... (consecutive threads read consecutive outputs: coalesced), then one thread per output adds
// the slices in order.  fp64, fixed order.
__global__ void dice_combine_kernel(const float* __restrict__ partial, int nblk, int L,
                                    float* __restrict__ sums) {
  extern __shared__ double s_part[];                   // [nslice][3L]
  const int b = blockIdx.x, n3 = 3 * L;
  const int nslice = blockDim.x / n3;
  const int slice = threadIdx.x / n3, o = threadIdx.x - slice * n3;
  if (slice < nslice) {
    double s = 0.0;
    for (int k = slice; k < nblk; k += nslice) s += (double)partial[((int64_t)b * nblk + k) * n3 + o];
    s_part[slice * n3 + o] = s;
  }
  __syncthreads();
  if (threadIdx.x < n3) {
    double s = 0.0;
    for (int sl = 0; sl < nslice; ++sl) s += s_part[sl * n3 + threadIdx.x];
    const int kind = threadIdx.x / L, l = threadIdx.x - kind * L;
    sums[((int64_t)b * L + l) * 3 + kind] = (float)s;
  }
}

static int launch_dice_combine(const float* partial, int nblk, int B, int L, float* sums, cudaStream_t st) {
  if (3 * L <= 1024) {
    const int nslice = 1024 / (3 * L);
    dice_combine_kernel<<<B, 1024, (size_t)nslice * 3 * L * sizeof(double), st>>>(partial, nblk, L, sums);
  } else {
    dice_combine_serial_kernel<<<B, 128, 0, st>>>(partial, nblk, L, sums);
  }
  return check_launch("dice_combine_kernel");
}

__global__ void dice_finalize_kernel(const float* __restrict__ sums, int n, float eps,
                                     float* __restrict__ dice) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float top = __fmul_rn(2.0f, sums[i * 3 + 0]);                       // metrics.py:476
  const float bottom = __fadd_rn(sums[i * 3 + 1], sums[i * 3 + 2]);         // :477
  float d;
  if (eps > 0.f) d = __fdiv_rn(__fadd_rn(top, eps), __fadd_rn(bottom, eps));   // :478-480
  else d = (bottom != 0.f) ? __fdiv_rn(top, bottom) : 0.f;                  // divide_no_nan :482
  dice[i] = d;
}

__global__ void __launch_bounds__(kThreads)
argmax_kernel(const float* __restrict__ x, int64_t n, int L, int32_t* __restrict__ idx) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const float* row = x + r * L;
    float best = row[0];
    int bi = 0;
    for (int l = 1; l < L; ++l) { const float v = row[l]; if (v > best) { best = v; bi = l; } }
    idx[r] = bi;
  }
}

// ---------------------------------------------------------------------------------------
// categorical cross-entropy
// ---------------------------------------------------------------------------------------
struct CceArgs {
  const float* label_w;
  const float* sample_w;
  float* per_elem;
  int64_t n;
  int C;
  int from_logits;
  float smoothing;
};

// Q = C/4 lanes per row (a power of two <= 32, compile time: the group shuffles unroll, no loop counters, no branches):
// perfectly coalesced float4 streams; U rows per thread and pass, i.e. U independent pairs of streaming loads in flight
// per thread (a run-time q with one load pair per thread stalls on long-scoreboard waits and spends half of its
// instructions on the ALU pipe).
template <int Q>
__device__ __forceinline__ float group_sum_c(float v) {
#pragma unroll
  for (int o = Q >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int Q>
__device__ __forceinline__ float group_max_c(float v) {
#pragma unroll
  for (int o = Q >> 1; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <int Q, int U>
__global__ void __launch_bounds__(kThreads)
cce_vec4u_kernel(const float4* __restrict__ t4, const float4* __restrict__ p4, CceArgs a, float* __restrict__ partial) {
  __shared__ float s_red[kThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const int sub = lane & (Q - 1);
  constexpr int RPP = kThreads / Q;                      // rows per pass and sub-step
  float4 lw = make_float4(1.f, 1.f, 1.f, 1.f);
  if (a.label_w) lw = __ldg(reinterpret_cast<const float4*>(a.label_w) + sub);
  const float eps = 1e-7f, one_m_eps = __fsub_rn(1.0f, 1e-7f);
  const float sm_keep = __fsub_rn(1.0f, a.smoothing), sm_add = __fdiv_rn(a.smoothing, (float)a.C);
  float acc = 0.f;
  // block-uniform trip count: the group shuffles need every lane of the warp present
  for (int64_t r0 = (int64_t)blockIdx.x * (RPP * U); r0 < a.n; r0 += (int64_t)gridDim.x * (RPP * U)) {
    float4 t[U], p[U];
    int64_t r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      r[u] = r0 + u * RPP + tid / Q;
      t[u] = make_float4(0.f, 0.f, 0.f, 0.f); p[u] = make_float4(1.f, 1.f, 1.f, 1.f);
      if (r[u] < a.n) { t[u] = ld_stream_f4(t4 + r[u] * Q + sub); p[u] = ld_stream_f4(p4 + r[u] * Q + sub); }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float4 tt = t[u];
      const float4 pp = p[u];
      tt.x *= lw.x; tt.y *= lw.y; tt.z *= lw.z; tt.w *= lw.w;                   // metrics.py:648
      if (a.smoothing != 0.f) {
        tt.x = tt.x * sm_keep + sm_add; tt.y = tt.y * sm_keep + sm_add; tt.z = tt.z * sm_keep + sm_add; tt.w = tt.w * sm_keep + sm_add;
      }
      float l;
      if (!a.from_logits) {
        const float rs = __frcp_rn(group_sum_c<Q>((pp.x + pp.y) + (pp.z + pp.w)));
        const float a0 = fminf(fmaxf(pp.x * rs, eps), one_m_eps), a1 = fminf(fmaxf(pp.y * rs, eps), one_m_eps);
        const float a2 = fminf(fmaxf(pp.z * rs, eps), one_m_eps), a3 = fminf(fmaxf(pp.w * rs, eps), one_m_eps);
        // logf, not __logf: near q = 1 (a confident prediction) the loss term is log q itself, and __logf is only
        // accurate to an absolute 2^-21.41 there (6e-3 relative error at q = 0.99999, measured on H100)
        l = (tt.x * logf(a0) + tt.y * logf(a1)) + (tt.z * logf(a2) + tt.w * logf(a3));
      } else {
        const float m = group_max_c<Q>(fmaxf(fmaxf(pp.x, pp.y), fmaxf(pp.z, pp.w)));
        const float z0 = pp.x - m, z1 = pp.y - m, z2 = pp.z - m, z3 = pp.w - m;
        const float lse = logf(group_sum_c<Q>((expf(z0) + expf(z1)) + (expf(z2) + expf(z3))));
        l = (tt.x * (z0 - lse) + tt.y * (z1 - lse)) + (tt.z * (z2 - lse) + tt.w * (z3 - lse));
      }
      l = -group_sum_c<Q>(l);
      if (sub == 0 && r[u] < a.n) {
        if (a.sample_w) l *= __ldg(a.sample_w + r[u]);
        if (a.per_elem) a.per_elem[r[u]] = l;
        acc += l;
      }
    }
  }
  acc = warp_sum(acc);
  if (lane == 0) s_red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) s += s_red[i];
    partial[blockIdx.x] = s;
  }
}

// generic path: one thread per row, any C
__global__ void __launch_bounds__(kThreads)
cce_row_kernel(const float* __restrict__ t, const float* __restrict__ p, CceArgs a,
               float* __restrict__ partial) {
  __shared__ float s_red[kThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const float eps = 1e-7f, one_m_eps = __fsub_rn(1.0f, 1e-7f);
  const float sm_keep = __fsub_rn(1.0f, a.smoothing), sm_add = __fdiv_rn(a.smoothing, (float)a.C);
  float acc = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * kThreads + tid; r < a.n; r += (int64_t)gridDim.x * kThreads) {
    const float* tr = t + r * a.C;
    const float* pr = p + r * a.C;
    float l = 0.f;
    if (!a.from_logits) {
      float s = 0.f;
      for (int c = 0; c < a.C; ++c) s += pr[c];
      for (int c = 0; c < a.C; ++c) {
        float tv = tr[c] * (a.label_w ? __ldg(a.label_w + c) : 1.f);
        if (a.smoothing != 0.f) tv = tv * sm_keep + sm_add;
        l += tv * logf(fminf(fmaxf(__fdiv_rn(pr[c], s), eps), one_m_eps));
      }
    } else {
      float m = pr[0];
      for (int c = 1; c < a.C; ++c) m = fmaxf(m, pr[c]);
      float s = 0.f;
      for (int c = 0; c < a.C; ++c) s += expf(pr[c] - m);
      const float lse = logf(s);
      for (int c = 0; c < a.C; ++c) {
        float tv = tr[c] * (a.label_w ? __ldg(a.label_w + c) : 1.f);
        if (a.smoothing != 0.f) tv = tv * sm_keep + sm_add;
        l += tv * ((pr[c] - m) - lse);
      }
    }
    l = -l;
    if (a.sample_w) l *= __ldg(a.sample_w + r);
    if (a.per_elem) a.per_elem[r] = l;
    acc += l;
  }
  acc = warp_sum(acc);
  if (lane == 0) s_red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) s += s_red[i];
    partial[blockIdx.x] = s;
  }
}

__global__ void sum_partials_kernel(const float* __restrict__ partial, int n, float* __restrict__ out) {
  __shared__ double s[32];
  double v = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) v += (double)partial[i];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += s[i];
    out[0] = (float)tot;
  }
}

static int dice_blocks(int64_t work_items, int B) {
  // enough CTAs to fill the chip ~4 deep, bounded by the workspace
  int64_t want = ((int64_t)sm_count() * 8 + B - 1) / B;
  int64_t by_work = (work_items + 4095) / 4096;
  int64_t n = want < by_work ? want : by_work;
  if (n < 1) n = 1;
  if (n > kMaxBlocks) n = kMaxBlocks;
  return (int)n;
}

}  // namespace nrt

using namespace nrt;

extern "C" {

int64_t nrt_dice_workspace_bytes(int B, int L) {
  if (B < 1 || L < 1) return 0;
  return (int64_t)B * kMaxBlocks * 3 * L * (int64_t)sizeof(float);
}

int nrt_dice_sums_f32(const float* y_true, const float* y_pred, int B, int64_t V, int L, int64_t v0,
                      int64_t nv, int normalize, int check_limits, float* sums, int32_t* flag,
                      void* workspace, int64_t workspace_bytes, void* stream) {
  NRT_REQUIRE(y_true && y_pred && sums && workspace, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(!check_limits || flag, NRT_E_ARG, "check_limits needs a flag pointer");
  NRT_REQUIRE(B >= 1 && L >= 1 && V >= 0, NRT_E_ARG, "bad B/L/V");
  NRT_REQUIRE(v0 >= 0 && nv >= 0 && v0 + nv <= V, NRT_E_ARG, "voxel range [%lld,%lld) outside [0,%lld)",
              (long long)v0, (long long)(v0 + nv), (long long)V);
  NRT_REQUIRE(workspace_bytes >= nrt_dice_workspace_bytes(B, L), NRT_E_ARG, "workspace too small");
  NRT_REQUIRE(B <= 65535, NRT_E_SIZE, "B > 65535");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* partial = static_cast<float*>(workspace);
  int32_t* flg = flag;
  static int32_t* dummy = nullptr;
  (void)dummy;
  int nblk;
  const bool vec_ok = !normalize && (L % 4 == 0) && (L / 4) <= kThreads && aligned16(y_true) && aligned16(y_pred);
  if (vec_ok) {
    const int q = L / 4;
    const int nthr = kThreads / q * q;
    const int64_t n4 = nv * q;
    nblk = dice_blocks(n4, B);
    dim3 grid(nblk, B);
    dice_sums_vec4_kernel<4><<<grid, kThreads, 0, st>>>(reinterpret_cast<const float4*>(y_true),
                                                       reinterpret_cast<const float4*>(y_pred), V * q, v0 * q, n4, q,
                                                       nthr, check_limits, partial, flg);
  } else if (!normalize && L <= kThreads) {
    const int nthr = kThreads / L * L;
    const int64_t n = nv * L;
    nblk = dice_blocks(n / 4, B);
    dim3 grid(nblk, B);
    dice_sums_scalar_kernel<<<grid, kThreads, 0, st>>>(y_true, y_pred, V * L, v0 * L, n, L, nthr, check_limits, partial, flg);
  } else {
    NRT_REQUIRE((size_t)3 * L * sizeof(float) <= 48 * 1024, NRT_E_SIZE, "L = %d too large", L);
    nblk = dice_blocks(nv * L / 4, B);
    dim3 grid(nblk, B);
    dice_sums_voxel_kernel<<<grid, kThreads, 3 * L * sizeof(float), st>>>(y_true, y_pred, V, v0, nv, L, normalize,
                                                                          check_limits, partial, flg);
  }
  int rc = check_launch("dice_sums kernel");
  if (rc != NRT_OK) return rc;
  return launch_dice_combine(partial, nblk, B, L, sums, st);
}

int nrt_dice_label_sums_i32(const int32_t* t_lab, const int32_t* p_lab, int B, int64_t V, int L, int64_t v0,
                            int64_t nv, float* sums, void* workspace, int64_t workspace_bytes, void* stream) {
  NRT_REQUIRE(t_lab && p_lab && sums && workspace, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 1 && B <= 65535 && L >= 1 && V >= 0, NRT_E_ARG, "bad B/L/V");
  NRT_REQUIRE(v0 >= 0 && nv >= 0 && v0 + nv <= V, NRT_E_ARG, "voxel range outside [0,V)");
  NRT_REQUIRE(workspace_bytes >= nrt_dice_workspace_bytes(B, L), NRT_E_ARG, "workspace too small");
  NRT_REQUIRE((size_t)3 * L * sizeof(int) <= 48 * 1024, NRT_E_SIZE, "L = %d too large", L);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* partial = static_cast<float*>(workspace);
  const int nblk = dice_blocks(nv / 4, B);
  dim3 grid(nblk, B);
  dice_label_counts_kernel<<<grid, kThreads, 3 * L * sizeof(int), st>>>(t_lab, p_lab, V, v0, nv, L, partial);
  int rc = check_launch("dice_label_counts_kernel");
  if (rc != NRT_OK) return rc;
  return launch_dice_combine(partial, nblk, B, L, sums, st);
}

int nrt_argmax_f32(const float* x, int64_t n, int L, int32_t* idx, void* stream) {
  NRT_REQUIRE(x && idx, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(n >= 0 && L >= 1, NRT_E_ARG, "bad n/L");
  if (n == 0) return NRT_OK;
  const int grid = (int)imin64((n + kThreads - 1) / kThreads, (int64_t)sm_count() * 16);
  argmax_kernel<<<grid, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, n, L, idx);
  return check_launch("argmax_kernel");
}

int nrt_dice_finalize_f32(const float* sums, int B, int L, float laplace, float* dice, void* stream) {
  NRT_REQUIRE(sums && dice, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 1 && L >= 1, NRT_E_ARG, "bad B/L");
  const int n = B * L;
  dice_finalize_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(sums, n, laplace, dice);
  return check_launch("dice_finalize_kernel");
}

int64_t nrt_cce_workspace_bytes(void) { return (int64_t)kMaxBlocks * 4 * sizeof(float); }

int nrt_cce_f32(const float* y_true, const float* y_pred, const float* label_w, const float* sample_w,
                int64_t n, int C, int from_logits, float label_smoothing, float* per_elem, float* sum_out,
                void* workspace, int64_t workspace_bytes, void* stream) {
  NRT_REQUIRE(y_true && y_pred && sum_out && workspace, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(n >= 0 && C >= 1, NRT_E_ARG, "bad n/C");
  NRT_REQUIRE(workspace_bytes >= nrt_cce_workspace_bytes(), NRT_E_ARG, "workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* partial = static_cast<float*>(workspace);
  CceArgs a{label_w, sample_w, per_elem, n, C, from_logits, label_smoothing};
  const int q = C / 4;
  const bool vec_ok = (C % 4 == 0) && q <= 32 && (q & (q - 1)) == 0 && aligned16(y_true) && aligned16(y_pred) &&
                      (!label_w || aligned16(label_w));
  int grid;
  if (n == 0) {
    cudaMemsetAsync(sum_out, 0, sizeof(float), st);
    return check_launch("cce memset");
  }
  if (vec_ok) {
    constexpr int kU = 4;                                // rows per thread and pass
    const int rows_per_pass = kThreads / q * kU;
    grid = (int)imin64((n + rows_per_pass - 1) / rows_per_pass, (int64_t)min(kMaxBlocks * 4, sm_count() * 8));
    const float4* t4 = reinterpret_cast<const float4*>(y_true);
    const float4* p4 = reinterpret_cast<const float4*>(y_pred);
    switch (q) {
      case 1: cce_vec4u_kernel<1, kU><<<grid, kThreads, 0, st>>>(t4, p4, a, partial); break;
      case 2: cce_vec4u_kernel<2, kU><<<grid, kThreads, 0, st>>>(t4, p4, a, partial); break;
      case 4: cce_vec4u_kernel<4, kU><<<grid, kThreads, 0, st>>>(t4, p4, a, partial); break;
      case 8: cce_vec4u_kernel<8, kU><<<grid, kThreads, 0, st>>>(t4, p4, a, partial); break;
      case 16: cce_vec4u_kernel<16, kU><<<grid, kThreads, 0, st>>>(t4, p4, a, partial); break;
      default: cce_vec4u_kernel<32, kU><<<grid, kThreads, 0, st>>>(t4, p4, a, partial); break;
    }
  } else {
    grid = (int)imin64((n + kThreads - 1) / kThreads, (int64_t)min(kMaxBlocks * 4, sm_count() * 8));
    cce_row_kernel<<<grid, kThreads, 0, st>>>(y_true, y_pred, a, partial);
  }
  int rc = check_launch("cce kernel");
  if (rc != NRT_OK) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, grid, sum_out);
  return check_launch("sum_partials_kernel");
}

}  // extern "C"
