// nrt_synth.cu -- the label-to-image stages of the synthesis generator labels_to_image_new: per-label intensities
// with the bias field, min-max normalisation and gamma, the output label map (one-hot or remapped) and the crop
// window of RandomCrop.
//
// Reference: neurite/tf/models.py:1162-1282 (labels_to_image_new), neurite/tf/layers.py:446-519 (RandomCrop),
// neurite/tf/utils/utils.py:953-968 (minmax_norm).
//
// Label maps arrive as the fp32 output of the nearest-neighbour warp, [B, V] (one channel).  A voxel's label is
// int32(truncate(x)), as tf.cast.  The crop is a window [lo, hi) on one spatial axis, given as (L, inner): the
// voxel v of an item lies at (v / inner) % L on that axis; a voxel outside the window has label 0.  A LUT
// lookup with an index outside [0, n) gives 0, as TF's GPU gather does.
//
// Every product, sum and quotient below is rounded once (__f*_rn, no FMA contraction), in TF's order:
//   mean   u * (max - min) + min                          (tf.random.uniform with per-label bounds)
//   image  mean * expf(bias)                               (bias_func = tf.exp, then image *= bias)
//   norm   (x - mn) / (mx - mn), 0 where mx == mn          (tf.compat.v1.div_no_nan)
//   gamma  powf(norm, u * (hi - lo) + lo)
#include <type_traits>

#include "nrt_common.cuh"

namespace nrt {
namespace {

struct Crop {
  uint32_t L, inner, lo, hi;
};

__device__ __forceinline__ bool in_window(uint32_t v, const Crop& w) {
  const uint32_t a = (v / w.inner) % w.L;
  return a >= w.lo && a < w.hi;
}

__device__ __forceinline__ int lut_at(const int32_t* lut, int n, int i) { return (i >= 0 && i < n) ? lut[i] : 0; }

__device__ __forceinline__ int crop_label(const float* labels, uint32_t b, uint32_t V, uint32_t v, const Crop& w) {
  return in_window(v, w) ? __float2int_rz(__ldg(labels + (uint64_t)b * V + v)) : 0;
}

// ---- 1: label -> intensity [* expf(bias)], with block partials of max |image| ----
constexpr int kImThreads = 256;
constexpr int kImMaxBlocks = 1024;
// generation LUT entries held in shared memory: 48 KB without an opt-in, less the kernel's static partials
constexpr int kLutSmem = (48 * 1024 - (kImThreads / 32) * (int)sizeof(float)) / (int)sizeof(int32_t);

__global__ void __launch_bounds__(kImThreads) labels_to_image_kernel(
    const float* __restrict__ labels, uint32_t B, uint32_t V, int C, const Crop w, const int32_t* __restrict__ lut,
    int nlut, int N, const float* __restrict__ u, const float* __restrict__ mean_min,
    const float* __restrict__ mean_max, const float* __restrict__ bias, int apply_exp, float* __restrict__ image,
    float* __restrict__ mean_out, float* __restrict__ bias_out, float* __restrict__ partial) {
  extern __shared__ int32_t s_lut[];
  const bool smem = nlut <= kLutSmem;
  if (smem)
    for (int i = threadIdx.x; i < nlut; i += kImThreads) s_lut[i] = __ldg(lut + i);
  __syncthreads();
  const int32_t* tab = smem ? s_lut : lut;
  float amax = 0.f;
  const uint64_t total = (uint64_t)B * V;
  for (uint64_t e = (uint64_t)blockIdx.x * kImThreads + threadIdx.x; e < total; e += (uint64_t)gridDim.x * kImThreads) {
    const uint32_t b = (uint32_t)(e / V), v = (uint32_t)(e - (uint64_t)b * V);
    const int idx = lut_at(tab, nlut, crop_label(labels, b, V, v, w));
    for (int c = 0; c < C; ++c) {
      const float lo = __ldg(mean_min + c * N + idx), hi = __ldg(mean_max + c * N + idx);
      const float m = __fadd_rn(__fmul_rn(__ldg(u + ((uint64_t)b * C + c) * N + idx), __fsub_rn(hi, lo)), lo);
      const uint64_t o = e * C + c;
      float x = m;
      if (bias) {
        float f = ld_stream_f(bias + o);
        if (apply_exp) f = expf(f);
        if (bias_out) bias_out[o] = f;
        x = __fmul_rn(m, f);
        if (mean_out) mean_out[o] = m;
      }
      image[o] = x;
      amax = fmaxf(amax, fabsf(x));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  __shared__ float sh[kImThreads / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = amax;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < kImThreads / 32; ++i) amax = fmaxf(amax, sh[i]);
    partial[blockIdx.x] = amax;
  }
}

// one warp: the max of the block partials, in a fixed order
__global__ void absmax_final_kernel(const float* __restrict__ partial, int nb, float* __restrict__ out) {
  float m = 0.f;
  for (int i = threadIdx.x; i < nb; i += 32) m = fmaxf(m, partial[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (threadIdx.x == 0) *out = m;
}

// ---- 3: (x - mn) / (mx - mn) with the per-item min / max of nrt_stats.cu, and / or the gamma power ----
__global__ void __launch_bounds__(256) norm_gamma_kernel(const float* __restrict__ x, int items, int64_t n, int C,
                                                         const float2* __restrict__ mnmx,
                                                         const float* __restrict__ gamma_u, float g_lo, float g_hi,
                                                         float* __restrict__ out) {
  const int64_t total = (int64_t)items * n;
  const float gd = __fsub_rn(g_hi, g_lo);
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256) {
    const int item = (int)(e / n);
    float y = ld_stream_f(x + e);
    if (mnmx) {
      const float2 m = mnmx[item];
      const float d = __fsub_rn(m.y, m.x);
      y = d == 0.f ? 0.f : __fdiv_rn(__fsub_rn(y, m.x), d);
    }
    if (gamma_u) {
      const int c = (int)(e % C);
      const float g = __fadd_rn(__fmul_rn(__ldg(gamma_u + (int64_t)item * C + c), gd), g_lo);
      y = powf(y, g);
    }
    st_stream_f(out + e, y);
  }
}

// ---- 4: crop + output LUT -> one-hot [B, V, M] (fp32, 16-byte stores) or label map [B, V] (int32) ----
__device__ __forceinline__ int out_label(const float* labels, uint32_t b, uint32_t V, uint32_t v, const Crop& w,
                                         const int32_t* lut, int nlut) {
  const int l = crop_label(labels, b, V, v, w);
  return lut ? lut_at(lut, nlut, l) : l;
}

// Thread q writes out[4q .. 4q+3] of the flat [B * V * M] one-hot: the row of voxel e / M, column e % M.
// The label of a voxel is read by the ceil(M / 4) threads that write its row (L1 hits after the first).
__global__ void __launch_bounds__(256) one_hot_kernel(const float* __restrict__ labels, uint32_t B, uint32_t V,
                                                      const Crop w, const int32_t* __restrict__ lut, int nlut, int M,
                                                      float* __restrict__ out, int vec) {
  const uint64_t total = (uint64_t)B * V * M, nq = (total + 3) / 4;
  for (uint64_t q = (uint64_t)blockIdx.x * 256 + threadIdx.x; q < nq; q += (uint64_t)gridDim.x * 256) {
    const uint64_t e0 = q * 4;
    uint64_t bv = e0 / (uint32_t)M;
    int c = (int)(e0 - bv * (uint32_t)M);
    uint32_t b = (uint32_t)(bv / V), v = (uint32_t)(bv - (uint64_t)b * V);
    int idx = out_label(labels, b, V, v, w, lut, nlut);
    float r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      r[k] = c == idx ? 1.f : 0.f;
      if (++c == M && k < 3) {
        c = 0;
        if (++v == V) { v = 0; ++b; }
        if (b < B) idx = out_label(labels, b, V, v, w, lut, nlut);
      }
    }
    if (vec && e0 + 3 < total) {
      st_stream_f4(reinterpret_cast<float4*>(out + e0), make_float4(r[0], r[1], r[2], r[3]));
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (e0 + k < total) out[e0 + k] = r[k];
    }
  }
}

__global__ void __launch_bounds__(256) label_map_kernel(const float* __restrict__ labels, uint32_t B, uint32_t V,
                                                        const Crop w, const int32_t* __restrict__ lut, int nlut,
                                                        int32_t* __restrict__ out) {
  const uint64_t total = (uint64_t)B * V;
  for (uint64_t e = (uint64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (uint64_t)gridDim.x * 256) {
    const uint32_t b = (uint32_t)(e / V), v = (uint32_t)(e - (uint64_t)b * V);
    out[e] = out_label(labels, b, V, v, w, lut, nlut);
  }
}

// ---- 5: x * mask on [outer, L, inner], mask 1 on [lo, hi) along L (RandomCrop) ----
template <typename T>
__global__ void __launch_bounds__(256) crop_window_kernel(const T* __restrict__ x, int64_t outer, int64_t L,
                                                          int64_t inner, int64_t lo, int64_t hi, T* __restrict__ out) {
  const int64_t total = outer * L * inner;
  for (int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (int64_t)gridDim.x * 256) {
    const int64_t a = (e / inner) % L;
    const bool keep = a >= lo && a < hi;
    if constexpr (std::is_same<T, float>::value) out[e] = __fmul_rn(x[e], keep ? 1.f : 0.f);   // x * mask
    else out[e] = keep ? x[e] : T(0);
  }
}

inline int grid_for(int64_t work, int per_block) {
  return (int)imin64((work + per_block - 1) / per_block, (int64_t)sm_count() * 16);
}

int make_crop(int64_t crop_L, int64_t crop_inner, int64_t crop_lo, int64_t crop_hi, int64_t V, Crop* w) {
  NRT_REQUIRE(crop_L >= 1 && crop_inner >= 1 && crop_L * crop_inner <= V && V % (crop_L * crop_inner) == 0, NRT_E_ARG,
              "crop axis (L = %lld, inner = %lld) does not divide an item of %lld voxels", (long long)crop_L,
              (long long)crop_inner, (long long)V);
  NRT_REQUIRE(crop_lo >= 0 && crop_lo <= crop_hi && crop_hi <= crop_L, NRT_E_ARG, "crop window [%lld, %lld) outside [0, %lld]",
              (long long)crop_lo, (long long)crop_hi, (long long)crop_L);
  *w = Crop{(uint32_t)crop_L, (uint32_t)crop_inner, (uint32_t)crop_lo, (uint32_t)crop_hi};
  return NRT_OK;
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int64_t nrt_labels_to_image_workspace_bytes(void) { return (int64_t)kImMaxBlocks * (int64_t)sizeof(float); }

int nrt_labels_to_image_f32(const float* labels, int B, int64_t V, int C, int64_t crop_L, int64_t crop_inner,
                            int64_t crop_lo, int64_t crop_hi, const int32_t* gen_lut, int nlut, int N, const float* u,
                            const float* mean_min, const float* mean_max, const float* bias, int apply_exp,
                            float* image, float* mean_out, float* bias_out, float* absmax, void* workspace,
                            int64_t workspace_bytes, void* stream) {
  NRT_REQUIRE(labels && gen_lut && u && mean_min && mean_max && image && absmax && workspace, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 1 && V >= 1 && C >= 1 && nlut >= 1 && N >= 1, NRT_E_ARG, "bad B / V / C / LUT / label count");
  NRT_REQUIRE((int64_t)B * V <= 4294967295LL && (int64_t)B * V * C <= ((int64_t)1 << 40), NRT_E_SIZE, "label map too large");
  NRT_REQUIRE(!(mean_out || bias_out) || bias, NRT_E_ARG, "mean / bias outputs need a bias field");
  NRT_REQUIRE(workspace_bytes >= nrt_labels_to_image_workspace_bytes(), NRT_E_ARG, "workspace too small");
  Crop w;
  if (int rc = make_crop(crop_L, crop_inner, crop_lo, crop_hi, V, &w)) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nb = (int)imin64(grid_for((int64_t)B * V, kImThreads), kImMaxBlocks);
  const size_t smem = nlut <= kLutSmem ? (size_t)nlut * sizeof(int32_t) : 0;
  float* partial = static_cast<float*>(workspace);
  labels_to_image_kernel<<<nb, kImThreads, smem, st>>>(labels, (uint32_t)B, (uint32_t)V, C, w, gen_lut, nlut, N, u,
                                                       mean_min, mean_max, bias, apply_exp, image, mean_out, bias_out,
                                                       partial);
  if (int rc = check_launch("labels_to_image_kernel")) return rc;
  absmax_final_kernel<<<1, 32, 0, st>>>(partial, nb, absmax);
  return check_launch("absmax_final_kernel");
}

int nrt_norm_gamma_f32(const float* x, int items, int64_t n, int C, const float* mnmx, const float* gamma_u,
                       float gamma_lo, float gamma_hi, float* out, void* stream) {
  NRT_REQUIRE(x && out && (mnmx || gamma_u), NRT_E_ARG, "null pointer");
  NRT_REQUIRE(items >= 1 && n >= 1 && C >= 1 && n % C == 0, NRT_E_ARG, "bad items / n / C");
  const int64_t total = (int64_t)items * n;
  norm_gamma_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, items, n, C, reinterpret_cast<const float2*>(mnmx), gamma_u, gamma_lo, gamma_hi, out);
  return check_launch("norm_gamma_kernel");
}

int nrt_label_map_f32(const float* labels, int B, int64_t V, int64_t crop_L, int64_t crop_inner, int64_t crop_lo,
                      int64_t crop_hi, const int32_t* lut, int nlut, int M, float* out, void* stream) {
  NRT_REQUIRE(labels && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 1 && V >= 1 && M >= 1 && (!lut || nlut >= 1), NRT_E_ARG, "bad B / V / M / LUT");
  NRT_REQUIRE((int64_t)B * V <= 4294967295LL && (int64_t)B * V * M <= ((int64_t)1 << 40), NRT_E_SIZE,
              "one-hot map too large");
  Crop w;
  if (int rc = make_crop(crop_L, crop_inner, crop_lo, crop_hi, V, &w)) return rc;
  const int64_t nq = ((int64_t)B * V * M + 3) / 4;
  one_hot_kernel<<<grid_for(nq, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      labels, (uint32_t)B, (uint32_t)V, w, lut, nlut, M, out, aligned16(out) ? 1 : 0);
  return check_launch("one_hot_kernel");
}

int nrt_label_map_i32(const float* labels, int B, int64_t V, int64_t crop_L, int64_t crop_inner, int64_t crop_lo,
                      int64_t crop_hi, const int32_t* lut, int nlut, int32_t* out, void* stream) {
  NRT_REQUIRE(labels && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 1 && V >= 1 && (!lut || nlut >= 1), NRT_E_ARG, "bad B / V / LUT");
  NRT_REQUIRE((int64_t)B * V <= 4294967295LL, NRT_E_SIZE, "label map too large");
  Crop w;
  if (int rc = make_crop(crop_L, crop_inner, crop_lo, crop_hi, V, &w)) return rc;
  label_map_kernel<<<grid_for((int64_t)B * V, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      labels, (uint32_t)B, (uint32_t)V, w, lut, nlut, out);
  return check_launch("label_map_kernel");
}

int nrt_crop_window_f32(const float* x, int64_t outer, int64_t L, int64_t inner, int64_t lo, int64_t hi, float* out,
                        void* stream) {
  NRT_REQUIRE(x && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(outer >= 0 && L >= 0 && inner >= 0 && lo >= 0 && lo <= hi && hi <= L, NRT_E_ARG, "bad crop window");
  const int64_t total = outer * L * inner;
  if (total == 0) return NRT_OK;
  crop_window_kernel<float><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, outer, L, inner,
                                                                                                  lo, hi, out);
  return check_launch("crop_window_kernel<float>");
}

int nrt_crop_window_i32(const int32_t* x, int64_t outer, int64_t L, int64_t inner, int64_t lo, int64_t hi,
                        int32_t* out, void* stream) {
  NRT_REQUIRE(x && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(outer >= 0 && L >= 0 && inner >= 0 && lo >= 0 && lo <= hi && hi <= L, NRT_E_ARG, "bad crop window");
  const int64_t total = outer * L * inner;
  if (total == 0) return NRT_OK;
  crop_window_kernel<int32_t><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, outer, L, inner,
                                                                                                    lo, hi, out);
  return check_launch("crop_window_kernel<int>");
}

}  // extern "C"
