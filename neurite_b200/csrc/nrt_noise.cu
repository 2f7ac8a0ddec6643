// nrt_noise.cu -- the noise fields of the synthesis generator: a counter-based Philox4x32-10 stream (uniform SD
// tables, normal noise scaled by a broadcast SD table) and the mean over Perlin levels.  The per-item statistics
// the fields are rescaled by are in nrt_stats.cu.
//
// Reference: neurite/tf/utils/augment.py:65-218 (random_blur_rescale, draw_perlin_full), neurite/tf/layers.py:
// 2305-2508 (GaussianNoise, PerlinNoise).  TF's random stream cannot be reproduced outside TF; this one is defined
// here and restated in numpy by oracle/noise.py.
//
// Generator.  Philox4x32-10 (Salmon et al., SC'11) with the 64-bit key {key_lo, key_hi} and the 128-bit counter
// {j_lo, j_hi, 0, 0} yields four 32-bit words w[0..3] for block j; element i of a draw takes word i % 4 of block
// i / 4.  So a value depends on (key, i) only, never on the launch geometry: the first n values of a longer draw
// are the values of an n-element draw.
//   integer -> float:  u = ((w >> 8) + 1) * 2^-24, exact in fp32, in (0, 1] (log(u) is finite).
//   uniform:           lo + (hi - lo) * u, with hi - lo, the product and the sum each rounded once (no FMA), as
//                      TF's `rnd * (maxval - minval) + minval`; bit-exact to the numpy restatement.
//   normal (Box-Muller on the pairs (w0, w1) and (w2, w3)):
//                      r = sqrtf(-2 * logf(u_even)), (s, c) = sincospif(2 * u_odd),
//                      z_even = r * c, z_odd = r * s.
//                      logf and sincospif are the accurate CUDA functions (1 ulp each, CUDA Programming Guide,
//                      mathematical functions), sqrtf is correctly rounded and 2 * u is exact.  So
//                      |z - z_exact| <= 3 * 2^-23 * |z| against Box-Muller evaluated exactly on the same u (log
//                      2^-23 relative, halved by the root, plus the root's rounding 2^-24; cos / sin 2^-23; the
//                      product 2^-24: 2.5 * 2^-23).
//                      out = z * sd[t] (* scale) (+ x[i]): each product / sum rounded once.
#include "nrt_common.cuh"

namespace nrt {
namespace {

constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u;
constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u;

__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1) {
  uint32_t x0 = c0, x1 = c1, x2 = 0u, x3 = 0u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(kPhiloxM0, x0), lo0 = kPhiloxM0 * x0;
    const uint32_t hi1 = __umulhi(kPhiloxM1, x2), lo1 = kPhiloxM1 * x2;
    const uint32_t y0 = hi1 ^ x1 ^ k0, y2 = hi0 ^ x3 ^ k1;
    x0 = y0; x1 = lo1; x2 = y2; x3 = lo0;
    k0 += kPhiloxW0; k1 += kPhiloxW1;
  }
  return make_uint4(x0, x1, x2, x3);
}

__device__ __forceinline__ float u01(uint32_t w) { return (float)((w >> 8) + 1u) * 5.9604644775390625e-8f; }

// up to 5 collapsed dims of the draw (row-major), with the SD table's stride on each (0 = broadcast)
struct Bcast {
  uint32_t dims[5];
  uint32_t sd_stride[5];
  int nd;
};

__device__ __forceinline__ uint32_t table_index(uint32_t i, const Bcast& b) {
  uint32_t t = 0;
  for (int d = b.nd - 1; d > 0; --d) {
    const uint32_t q = i / b.dims[d];
    t += (i - q * b.dims[d]) * b.sd_stride[d];
    i = q;
  }
  return t + i * b.sd_stride[0];
}

__global__ void __launch_bounds__(256) philox_uniform_kernel(uint32_t k0, uint32_t k1, uint32_t n, float lo, float hi,
                                                             float* __restrict__ out) {
  const uint32_t j = blockIdx.x * 256u + threadIdx.x;
  if ((uint64_t)j * 4 >= n) return;
  const uint4 w = philox4x32_10(j, 0u, k0, k1);
  const float d = __fsub_rn(hi, lo);
  const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t i = j * 4u + q;
    if (i < n) out[i] = __fadd_rn(__fmul_rn(u01(ww[q]), d), lo);
  }
}

// the four standard normals of block j (Box-Muller on the word pairs)
__device__ __forceinline__ void philox_normal4(uint32_t j, uint32_t k0, uint32_t k1, float z[4]) {
  const uint4 w = philox4x32_10(j, 0u, k0, k1);
  const float r0 = sqrtf(-2.f * logf(u01(w.x))), r1 = sqrtf(-2.f * logf(u01(w.z)));
  float s0, c0, s1, c1;
  sincospif(2.f * u01(w.y), &s0, &c0);
  sincospif(2.f * u01(w.w), &s1, &c1);
  z[0] = __fmul_rn(r0, c0); z[1] = __fmul_rn(r0, s0);
  z[2] = __fmul_rn(r1, c1); z[3] = __fmul_rn(r1, s1);
}

__global__ void __launch_bounds__(256) philox_normal_kernel(uint32_t k0, uint32_t k1, uint32_t n, const Bcast b,
                                                            const float* __restrict__ sd,
                                                            const float* __restrict__ scale,
                                                            const float* __restrict__ x, float* __restrict__ out,
                                                            int vec) {
  const uint32_t j = blockIdx.x * 256u + threadIdx.x;
  if ((uint64_t)j * 4 >= n) return;
  float z[4];
  philox_normal4(j, k0, k1, z);
  const float sc = scale ? __ldg(scale) : 1.f;
  const uint32_t i0 = j * 4u;
  float v[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float s = __ldg(sd + table_index(min(i0 + q, n - 1), b));
    if (scale) s = __fmul_rn(s, sc);
    v[q] = __fmul_rn(z[q], s);
  }
  if (vec && i0 + 3 < n) {                              // 16-byte aligned x / out, whole block in range
    if (x) {
      const float4 xv = ld_stream_f4(reinterpret_cast<const float4*>(x + i0));
      v[0] = __fadd_rn(xv.x, v[0]); v[1] = __fadd_rn(xv.y, v[1]);
      v[2] = __fadd_rn(xv.z, v[2]); v[3] = __fadd_rn(xv.w, v[3]);
    }
    st_stream_f4(reinterpret_cast<float4*>(out + i0), make_float4(v[0], v[1], v[2], v[3]));
    return;
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t i = i0 + q;
    if (i < n) out[i] = x ? __fadd_rn(x[i], v[q]) : v[q];
  }
}

// GaussianNoise of the generator fused with its background clearing (models.py:1219-1231) on x [B, V, C]:
// out[i] = (x[i] + z_i * (sd[b, c] * scale)) * keep, keep = 0 where label(b, v) == 0 and bg_u[b] < zb, else 1.
// z_i is element i of the same draw as philox_normal_kernel with shape [B, V, C] and the SD table [B, 1, C].
// label(b, v) = int32(labels[b, v]) inside the crop window (v / crop_inner) % crop_L in [crop_lo, crop_hi), else 0.
__global__ void __launch_bounds__(256) philox_normal_background_kernel(
    uint32_t k0, uint32_t k1, uint32_t V, uint32_t C, uint32_t n, const float* __restrict__ sd,
    const float* __restrict__ scale, const float* __restrict__ x, const float* __restrict__ labels, uint32_t crop_L,
    uint32_t crop_inner, uint32_t crop_lo, uint32_t crop_hi, const float* __restrict__ bg_u, float zb,
    float* __restrict__ out) {
  const uint32_t j = blockIdx.x * 256u + threadIdx.x;
  if ((uint64_t)j * 4 >= n) return;
  float z[4];
  philox_normal4(j, k0, k1, z);
  const float sc = __ldg(scale);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t i = j * 4u + q;
    if (i >= n) break;
    const uint32_t bv = i / C, c = i - bv * C, b = bv / V, v = bv - b * V;
    const float s = __fmul_rn(__ldg(sd + b * C + c), sc);
    const float y = __fadd_rn(x[i], __fmul_rn(z[q], s));
    const uint32_t a = (v / crop_inner) % crop_L;
    const int lab = (a >= crop_lo && a < crop_hi) ? __float2int_rz(__ldg(labels + bv)) : 0;
    const bool clear = lab == 0 && __ldg(bg_u + b) < zb;
    out[i] = __fmul_rn(y, clear ? 0.f : 1.f);
  }
}

// out[g, i] = (sum_l x[l, g, i] * divide_no_nan(before[l*G + g], after[l*G + g])) / L, levels in order
__global__ void __launch_bounds__(256) level_combine_kernel(const float* __restrict__ x, int L, int G, int64_t m,
                                                            const float* __restrict__ before,
                                                            const float* __restrict__ after, float* __restrict__ out) {
  const int64_t total = (int64_t)G * m, level_stride = total;
  const float fl = (float)L;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(e / m);
    float acc = 0.f;
    for (int l = 0; l < L; ++l) {
      const float a = __ldg(after + l * G + g);
      const float r = a != 0.f ? __fdiv_rn(__ldg(before + l * G + g), a) : 0.f;
      acc = __fadd_rn(acc, __fmul_rn(ld_stream_f(x + l * level_stride + e), r));
    }
    out[e] = __fdiv_rn(acc, fl);
  }
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int nrt_philox_uniform_f32(uint64_t key, int64_t n, float lo, float hi, float* out, void* stream) {
  NRT_REQUIRE(out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(n >= 0, NRT_E_ARG, "bad n");
  NRT_REQUIRE(n <= 2147483647LL, NRT_E_SIZE, "draw of %lld elements > 2^31-1", (long long)n);
  if (n == 0) return NRT_OK;
  const unsigned blocks = (unsigned)((n + 1023) / 1024);
  philox_uniform_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      (uint32_t)key, (uint32_t)(key >> 32), (uint32_t)n, lo, hi, out);
  return check_launch("philox_uniform_kernel");
}

int nrt_philox_normal_f32(uint64_t key, const int32_t* shape, const int32_t* sd_shape, int ndim, const float* sd,
                          const float* sd_scale, const float* x, float* out, void* stream) {
  NRT_REQUIRE(shape && sd_shape && sd && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(ndim >= 1 && ndim <= 5, NRT_E_ARG, "ndim = %d outside 1..5", ndim);
  NRT_REQUIRE(!x || x != out, NRT_E_ARG, "in-place noise is not supported");
  int64_t n = 1;
  for (int d = 0; d < ndim; ++d) {
    NRT_REQUIRE(shape[d] >= 0, NRT_E_ARG, "negative extent");
    NRT_REQUIRE(sd_shape[d] == shape[d] || sd_shape[d] == 1, NRT_E_ARG,
                "SD table extent %d does not broadcast to %d on dim %d", sd_shape[d], shape[d], d);
    n *= shape[d];
  }
  NRT_REQUIRE(n <= 2147483647LL, NRT_E_SIZE, "draw of %lld elements > 2^31-1", (long long)n);
  if (n == 0) return NRT_OK;
  // collapse neighbouring dims that are both drawn along or both broadcast; drop extent-1 dims
  Bcast b{};
  b.nd = 0;
  uint32_t tstride = 1;
  uint32_t st[5];
  for (int d = ndim - 1; d >= 0; --d) { st[d] = sd_shape[d] == 1 ? 0u : tstride; tstride *= (uint32_t)sd_shape[d]; }
  uint32_t cd[5], cs[5];
  int nc = 0;
  for (int d = 0; d < ndim; ++d) {
    if (shape[d] == 1) continue;
    if (nc > 0 && ((cs[nc - 1] == 0) == (st[d] == 0))) {
      cd[nc - 1] *= (uint32_t)shape[d];
      if (st[d]) cs[nc - 1] = st[d];
    } else {
      cd[nc] = (uint32_t)shape[d]; cs[nc] = st[d]; ++nc;
    }
  }
  if (nc == 0) { cd[0] = 1; cs[0] = 0; nc = 1; }
  for (int d = 0; d < nc; ++d) { b.dims[d] = cd[d]; b.sd_stride[d] = cs[d]; }
  b.nd = nc;
  const int vec = aligned16(out) && (!x || aligned16(x));
  const unsigned blocks = (unsigned)((n + 1023) / 1024);
  philox_normal_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      (uint32_t)key, (uint32_t)(key >> 32), (uint32_t)n, b, sd, sd_scale, x, out, vec);
  return check_launch("philox_normal_kernel");
}

int nrt_philox_normal_background_f32(uint64_t key, int B, int64_t V, int C, const float* sd, const float* sd_scale,
                                     const float* x, const float* labels, int64_t crop_L, int64_t crop_inner,
                                     int64_t crop_lo, int64_t crop_hi, const float* bg_u, float zero_background,
                                     float* out, void* stream) {
  NRT_REQUIRE(sd && sd_scale && x && labels && bg_u && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(x != out, NRT_E_ARG, "in-place noise is not supported");
  NRT_REQUIRE(B >= 1 && V >= 1 && C >= 1, NRT_E_ARG, "bad B / V / C");
  NRT_REQUIRE(crop_L >= 1 && crop_inner >= 1 && V % (crop_L * crop_inner) == 0 && crop_lo >= 0 && crop_lo <= crop_hi &&
                  crop_hi <= crop_L, NRT_E_ARG, "bad crop window");
  const int64_t n = (int64_t)B * V * C;
  NRT_REQUIRE(n <= 2147483647LL, NRT_E_SIZE, "draw of %lld elements > 2^31-1", (long long)n);
  const unsigned blocks = (unsigned)((n + 1023) / 1024);
  philox_normal_background_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      (uint32_t)key, (uint32_t)(key >> 32), (uint32_t)V, (uint32_t)C, (uint32_t)n, sd, sd_scale, x, labels,
      (uint32_t)crop_L, (uint32_t)crop_inner, (uint32_t)crop_lo, (uint32_t)crop_hi, bg_u, zero_background, out);
  return check_launch("philox_normal_background_kernel");
}

int nrt_level_combine_f32(const float* x, int L, int G, int64_t m, const float* before, const float* after,
                          float* out, void* stream) {
  NRT_REQUIRE(x && before && after && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(L >= 1 && G >= 1 && m >= 0, NRT_E_ARG, "bad L/G/m");
  const int64_t total = (int64_t)G * m;
  if (total == 0) return NRT_OK;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 16);
  level_combine_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, L, G, m, before, after, out);
  return check_launch("level_combine_kernel");
}

}  // extern "C"
