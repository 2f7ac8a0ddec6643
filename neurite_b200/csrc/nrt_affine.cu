// nrt_affine.cu -- the label warp of labels_to_image_new in one pass: the per-item affine matrix, the optional
// deformation and the nearest-neighbour sample of the label map, fused.
//
// Reference: neurite/tf/models.py:1130-1160.  There the affine becomes a dense shift (AffineToDenseShift), is
// composed with the deformation (ComposeTransform: d + interpn_linear(shift, grid + d)) and the labels are warped
// with nearest interpolation and fill 0 (SpatialTransformer).  This kernel gives the same bits without
// materialising either field: the shift is evaluated where it is needed, from the matrix rows held in registers.
//
// For an output voxel x of item b (integer coordinates on the out grid), every op is rounded once (__f*_rn, no
// FMA contraction):
//   s_i(c) = ((M_i0 c_0 + M_i1 c_1) + M_i2 c_2) + M_iN - c_i            the dense shift at an integer point c
//   t      = s(x)                                                        without a deformation
//   t      = d(x) + L(x + d(x))                                          with one: L is interpn's linear sample of
//            the field s on the out grid (clip, floor, corner order, prod_n weights, sum from 0: nrt_common.cuh
//            axis_linear), its corner values s evaluated at the clamped corners
//   loc    = x + t; label = labels[b, rint(loc) clipped to the in grid], 0 where any loc_i < 0 or > in_i - 1.
//
// Mapping: a thread owns 4 consecutive voxels of one row of the last axis.  With a row length that is a multiple
// of 4 (and 16-byte aligned buffers) it reads d as N float4 and writes one float4; otherwise it goes voxel by
// voxel.  The labels are gathered through the read-only cache: one item's map stays resident in L2.
#include "nrt_common.cuh"

namespace nrt {
namespace {

constexpr int kAffThreads = 256;

struct AffGeo {
  int I[3];           // label (in) grid; only the first N are used
  int O[3];           // out grid
  uint32_t rows;      // product of the out extents but the last
  uint32_t quads;     // ceil(O[N - 1] / 4)
  uint64_t vin, vout; // voxels per item
};

// s_i at an integer point (exact float coordinates), in the fixed order above
template <int N>
__device__ __forceinline__ float shift_at(const float (&m)[N][N + 1], int i, const float (&c)[N]) {
  float s = __fmul_rn(m[i][0], c[0]);
#pragma unroll
  for (int k = 1; k < N; ++k) s = __fadd_rn(s, __fmul_rn(m[i][k], c[k]));
  return __fsub_rn(__fadd_rn(s, m[i][N]), c[i]);
}

template <int N, bool HAS_D>
__device__ __forceinline__ float warp_voxel(const float* __restrict__ lab, const float (&m)[N][N + 1],
                                            const AffGeo& g, const float (&x)[N], const float (&dv)[N]) {
  float t[N];
  if (HAS_D) {
    Axis a[N];
#pragma unroll
    for (int k = 0; k < N; ++k) a[k] = axis_linear(__fadd_rn(x[k], dv[k]), (float)(g.O[k] - 1), g.O[k] - 1);
    float acc[N];
#pragma unroll
    for (int i = 0; i < N; ++i) acc[i] = 0.f;
#pragma unroll
    for (int corner = 0; corner < (1 << N); ++corner) {
      float c[N];
      float w = 0.f;
#pragma unroll
      for (int k = 0; k < N; ++k) {
        const int bit = (corner >> (N - 1 - k)) & 1;       // first axis = most significant
        c[k] = (float)(bit ? a[k].i1 : a[k].i0);
        const float wk = bit ? a[k].whi : a[k].wlo;
        w = (k == 0) ? wk : __fmul_rn(w, wk);              // prod_n: ((w0*w1)*w2)
      }
#pragma unroll
      for (int i = 0; i < N; ++i) acc[i] = __fadd_rn(acc[i], __fmul_rn(w, shift_at<N>(m, i, c)));
    }
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = __fadd_rn(dv[i], acc[i]);
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = shift_at<N>(m, i, x);
  }
  bool oob = false;
  uint64_t idx = 0;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const float loc = __fadd_rn(x[k], t[k]);
    oob = oob || (loc < 0.f) || (loc > (float)(g.I[k] - 1));
    idx = idx * (uint64_t)g.I[k] + (uint64_t)axis_nearest(loc, g.I[k] - 1);
  }
  return apply_fill(__ldg(lab + idx), oob, 0.f);
}

template <int N, bool HAS_D, bool VEC>
__global__ void __launch_bounds__(kAffThreads) warp_labels_affine_kernel(
    const float* __restrict__ labels, const float* __restrict__ mats, const float* __restrict__ def,
    float* __restrict__ out, const AffGeo g, uint32_t B) {
  const uint64_t per_item = (uint64_t)g.rows * g.quads;
  const uint64_t tid = (uint64_t)blockIdx.x * kAffThreads + threadIdx.x;
  if (tid >= per_item * B) return;
  const uint32_t b = (uint32_t)(tid / per_item);
  const uint64_t rem = tid - (uint64_t)b * per_item;
  const uint32_t row = (uint32_t)(rem / g.quads);
  const int x0 = (int)(rem - (uint64_t)row * g.quads) * 4;
  const int X = g.O[N - 1];

  float m[N][N + 1];
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int k = 0; k <= N; ++k) m[i][k] = __ldg(mats + (uint64_t)b * (N * (N + 1)) + i * (N + 1) + k);

  float x[N];
  if (N == 3) {
    x[0] = (float)(row / (uint32_t)g.O[1]);
    x[1 % N] = (float)(row % (uint32_t)g.O[1]);
  } else {
    x[0] = (float)row;
  }
  const uint64_t v0 = (uint64_t)b * g.vout + (uint64_t)row * X + x0;
  const float* lab = labels + (uint64_t)b * g.vin;

  float dv[4][N];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int k = 0; k < N; ++k) dv[j][k] = 0.f;
  if (HAS_D) {
    if (VEC) {
      float f[4 * N];
      const float4* p = reinterpret_cast<const float4*>(def + v0 * N);
#pragma unroll
      for (int q = 0; q < N; ++q) {
        const float4 r = ld_stream_f4(p + q);
        f[4 * q] = r.x; f[4 * q + 1] = r.y; f[4 * q + 2] = r.z; f[4 * q + 3] = r.w;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int k = 0; k < N; ++k) dv[j][k] = f[j * N + k];
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (x0 + j < X)
#pragma unroll
          for (int k = 0; k < N; ++k) dv[j][k] = ld_stream_f(def + (v0 + j) * N + k);
    }
  }

  float r[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (VEC || x0 + j < X) {
      x[N - 1] = (float)(x0 + j);
      r[j] = warp_voxel<N, HAS_D>(lab, m, g, x, dv[j]);
    }
  }
  if (VEC) {
    st_stream_f4(reinterpret_cast<float4*>(out + v0), make_float4(r[0], r[1], r[2], r[3]));
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (x0 + j < X) out[v0 + j] = r[j];
  }
}

template <int N>
int launch(const float* labels, const float* mats, const float* def, float* out, const AffGeo& g, uint32_t B,
           cudaStream_t st) {
  const uint64_t threads = (uint64_t)g.rows * g.quads * B;
  const unsigned blocks = (unsigned)((threads + kAffThreads - 1) / kAffThreads);
  const bool vec = g.O[N - 1] % 4 == 0 && aligned16(out) && (!def || aligned16(def));
  if (def) {
    if (vec) warp_labels_affine_kernel<N, true, true><<<blocks, kAffThreads, 0, st>>>(labels, mats, def, out, g, B);
    else warp_labels_affine_kernel<N, true, false><<<blocks, kAffThreads, 0, st>>>(labels, mats, def, out, g, B);
  } else {
    if (vec) warp_labels_affine_kernel<N, false, true><<<blocks, kAffThreads, 0, st>>>(labels, mats, def, out, g, B);
    else warp_labels_affine_kernel<N, false, false><<<blocks, kAffThreads, 0, st>>>(labels, mats, def, out, g, B);
  }
  return check_launch("warp_labels_affine_kernel");
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int nrt_warp_labels_affine_f32(const float* labels, const float* mats, const float* def, float* out, int B, int N,
                               const int32_t* in_shape, const int32_t* out_shape, void* stream) {
  NRT_REQUIRE(labels && mats && out && in_shape && out_shape, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(N == 2 || N == 3, NRT_E_ARG, "N = %d: the label warp is built for 2 and 3 dimensions", N);
  NRT_REQUIRE(B >= 1, NRT_E_ARG, "B = %d", B);
  AffGeo g{};
  g.vin = g.vout = 1;
  for (int k = 0; k < 3; ++k) g.I[k] = g.O[k] = 1;
  for (int k = 0; k < N; ++k) {
    NRT_REQUIRE(in_shape[k] >= 1 && out_shape[k] >= 1, NRT_E_ARG, "empty axis %d", k);
    g.I[k] = in_shape[k];
    g.O[k] = out_shape[k];
    g.vin *= (uint64_t)in_shape[k];
    g.vout *= (uint64_t)out_shape[k];
  }
  NRT_REQUIRE(g.vin <= 2147483647ULL && g.vout <= 2147483647ULL && (uint64_t)B * g.vout <= ((uint64_t)1 << 40),
              NRT_E_SIZE, "label map too large");
  g.rows = (uint32_t)(g.vout / (uint64_t)g.O[N - 1]);
  g.quads = (uint32_t)((g.O[N - 1] + 3) / 4);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return N == 3 ? launch<3>(labels, mats, def, out, g, (uint32_t)B, st)
                : launch<2>(labels, mats, def, out, g, (uint32_t)B, st);
}

}  // extern "C"
