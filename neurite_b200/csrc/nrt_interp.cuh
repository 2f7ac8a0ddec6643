// nrt_interp.cuh -- pieces of the interpolation kernels shared by nrt_interp.cu (gather and box-tile kernels)
// and nrt_warp_march.cu (z-marching ring kernel for multi-channel volumes): geometry structs, the reference's
// per-point corner arithmetic (utils.py:137-204), the box-relative axis setup and the tensor-map encoder.
#pragma once
#include <cuda.h>   // CUtensorMap (types only; the encode entry point is fetched at run time)

#include "nrt_common.cuh"

namespace nrt {

struct Geo {
  int S[5];        // full spatial extent of the source volume per axis (clip bounds); axes 3, 4: interpn with D = 4, 5 only
  int src_z0;      // global index of the first resident source plane (axis 0)
  int src_n0;      // resident source planes
  int C;
  int has_fill;
  float fill;
  int32_t* err;    // device flag: corner outside the resident planes
};

// flat row-major index over the RESIDENT source (src_n0, S1, S2), reference sub2ind2d
template <int D>
__device__ __forceinline__ int flat_index(const Geo& g, const int (&sub)[D]) {
  int ndx = sub[0];
#pragma unroll
  for (int d = 1; d < D; ++d) ndx = ndx * g.S[d] + sub[d];
  return ndx;
}

__device__ __forceinline__ int to_resident(const Geo& g, int i) {
  int l = i - g.src_z0;
  if (l < 0 || l >= g.src_n0) {
    if (g.err) atomicOr(g.err, 1);
    l = min(max(l, 0), g.src_n0 - 1);
  }
  return l;
}

template <int D>
__device__ __forceinline__ bool out_of_bounds(const Geo& g, const float (&loc)[D]) {
  bool oob = false;
#pragma unroll
  for (int d = 0; d < D; ++d) oob = oob || (loc[d] < 0.0f) || (loc[d] > (float)(g.S[d] - 1));
  return oob;
}

// Corner indices (flat, resident) and weights of one output point.
template <int D, int METHOD>
struct Corners {
  int idx[METHOD == NRT_LINEAR ? (1 << D) : 1];
  float w[METHOD == NRT_LINEAR ? (1 << D) : 1];
};

template <int D, int METHOD>
__device__ __forceinline__ void setup_point(const Geo& g, const float (&loc)[D], Corners<D, METHOD>& k) {
  if (METHOD == NRT_LINEAR) {
    Axis a[D];
#pragma unroll
    for (int d = 0; d < D; ++d) a[d] = axis_linear(loc[d], (float)(g.S[d] - 1), g.S[d] - 1);
    a[0].i0 = to_resident(g, a[0].i0);
    a[0].i1 = to_resident(g, a[0].i1);
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) {
      int sub[D];
      float w = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) {
        const int bit = (c >> (D - 1 - d)) & 1;          // first axis = most significant
        sub[d] = bit ? a[d].i1 : a[d].i0;
        const float wd = bit ? a[d].whi : a[d].wlo;
        w = (d == 0) ? wd : __fmul_rn(w, wd);             // prod_n: ((w0*w1)*w2)
      }
      k.idx[c] = flat_index<D>(g, sub);
      k.w[c] = w;
    }
  } else {
    int sub[D];
#pragma unroll
    for (int d = 0; d < D; ++d) sub[d] = axis_nearest(loc[d], g.S[d] - 1);
    sub[0] = to_resident(g, sub[0]);
    k.idx[0] = flat_index<D>(g, sub);
    k.w[0] = 1.f;
  }
}

// channels [c0, c0+VEC) of one point from precomputed corners -- global-memory gather
template <int D, int VEC, int METHOD>
__device__ __forceinline__ void gather_point(const float* __restrict__ vol, const Geo& g,
                                             const Corners<D, METHOD>& k, bool oob, int c0, float (&res)[VEC]) {
  if (METHOD == NRT_LINEAR) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) res[v] = 0.0f;
#pragma unroll
    for (int c = 0; c < (1 << D); ++c) {
      const size_t off = (size_t)k.idx[c] * g.C + c0;
      const float w = k.w[c];
      if (VEC == 4) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(vol + off));
        res[0] = __fadd_rn(res[0], __fmul_rn(w, q.x));
        res[1 % VEC] = __fadd_rn(res[1 % VEC], __fmul_rn(w, q.y));
        res[2 % VEC] = __fadd_rn(res[2 % VEC], __fmul_rn(w, q.z));
        res[3 % VEC] = __fadd_rn(res[3 % VEC], __fmul_rn(w, q.w));
      } else {
        res[0] = __fadd_rn(res[0], __fmul_rn(w, __ldg(vol + off)));
      }
    }
  } else {
    const size_t off = (size_t)k.idx[0] * g.C + c0;
    if (VEC == 4) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(vol + off));
      res[0] = q.x; res[1 % VEC] = q.y; res[2 % VEC] = q.z; res[3 % VEC] = q.w;
    } else {
      res[0] = __ldg(vol + off);
    }
  }
  if (g.has_fill) {
#pragma unroll
    for (int v = 0; v < VEC; ++v) res[v] = apply_fill(res[v], oob, g.fill);
  }
}

// One output point: VEC == 4 -> this thread's 4-channel chunk [c0, c0+4);
//                   VEC == 1 -> all C channels (corner setup is done once per point).
template <int D, int VEC, int METHOD>
__device__ __forceinline__ void sample_store(const float* __restrict__ vol, const Geo& g,
                                             const float (&loc)[D], int c0, float* __restrict__ dst) {
  Corners<D, METHOD> k;
  setup_point<D, METHOD>(g, loc, k);
  const bool oob = g.has_fill ? out_of_bounds<D>(g, loc) : false;
  if (VEC == 4) {
    float r[VEC];
    gather_point<D, VEC, METHOD>(vol, g, k, oob, c0, r);
    *reinterpret_cast<float4*>(dst + c0) = make_float4(r[0], r[1 % VEC], r[2 % VEC], r[3 % VEC]);
  } else {
    for (int c = 0; c < g.C; ++c) {
      float r[VEC];
      gather_point<D, VEC, METHOD>(vol, g, k, oob, c, r);
      dst[c] = r[0];
    }
  }
}

// the same, split: corner weights once per voxel, accumulation once per channel
__device__ __forceinline__ void corner_weights(float wz0, float wz1, float wy0, float wy1, float wx0, float wx1,
                                               float (&k)[8]) {
  const float w00 = __fmul_rn(wz0, wy0), w01 = __fmul_rn(wz0, wy1);
  const float w10 = __fmul_rn(wz1, wy0), w11 = __fmul_rn(wz1, wy1);
  k[0] = __fmul_rn(w00, wx0); k[1] = __fmul_rn(w00, wx1); k[2] = __fmul_rn(w01, wx0); k[3] = __fmul_rn(w01, wx1);
  k[4] = __fmul_rn(w10, wx0); k[5] = __fmul_rn(w10, wx1); k[6] = __fmul_rn(w11, wx0); k[7] = __fmul_rn(w11, wx1);
}
__device__ __forceinline__ float acc8(const float (&k)[8], const float (&v)[8]) {
  float r = __fadd_rn(0.f, __fmul_rn(k[0], v[0]));
#pragma unroll
  for (int c = 1; c < 8; ++c) r = __fadd_rn(r, __fmul_rn(k[c], v[c]));
  return r;
}

__device__ __forceinline__ float fill_if_oob(const Geo& g, float res, float lz, float ly, float lx) {
  const bool oob = (lz < 0.f) | (lz > (float)(g.S[0] - 1)) | (ly < 0.f) | (ly > (float)(g.S[1] - 1)) |
                   (lx < 0.f) | (lx > (float)(g.S[2] - 1));
  return apply_fill(res, oob, g.fill);
}

// Per-axis corner setup against the staged box.
//   EDGE = false: the box does not overhang the volume on this axis, so a sample whose two
//     corners are in the box satisfies 0 <= loc < max: clip() is the identity, i1 = i0 + 1
//     and the second corner sits at a compile-time stride.
//   EDGE = true: the reference's clip / min(i0+1, max) is applied first; the second corner's
//     offset becomes a run-time 0-or-stride.
// `c0` is clamped into the box so the (unconditional) shared-memory loads are always legal;
// `ok` says whether they were the right addresses.
template <bool EDGE, int BDIM>
struct AxisBox {
  int c0;        // first corner, box-relative, clamped
  int d;         // (second corner - first corner) in elements of this axis (EDGE only)
  float wlo, whi;
  bool ok;
  __device__ __forceinline__ void setup(float loc, int o, int lo, int hi, int maxi) {
    if (!EDGE) {
      const int i0 = __float2int_rd(loc);
      const unsigned r = (unsigned)(i0 - o);
      const unsigned c = min(r, (unsigned)(BDIM - 2));
      ok = (c == r);
      c0 = (int)c;
      d = 1;
      wlo = __fsub_rn(__fadd_rn((float)i0, 1.f), loc);
    } else {
      const float x = fminf(fmaxf(loc, 0.f), (float)maxi);
      const int i0 = __float2int_rd(x);
      const int i1 = min(i0 + 1, maxi);
      ok = (i0 >= lo) & (i1 <= hi);
      d = i1 - i0;                                   // 0 at the volume's far edge, else 1
      c0 = min(max(i0 - o, 0), BDIM - 1 - d);        // c0 + d stays inside the box
      wlo = __fsub_rn((float)i1, x);
    }
    whi = __fsub_rn(1.f, wlo);
  }
};

template <bool EDGE, int BDIM>
__device__ __forceinline__ int nearest_box(float loc, int o, int lo, int hi, int maxi, bool& ok) {
  const int i = EDGE ? axis_nearest(loc, maxi) : __float2int_rn(loc);
  if (EDGE) {
    ok = ok & (i >= lo) & (i <= hi);
    return min(max(i - o, 0), BDIM - 1);
  }
  const unsigned r = (unsigned)(i - o);
  const unsigned c = min(r, (unsigned)(BDIM - 1));
  ok = ok & (c == r);
  return (int)c;
}

struct BoxBounds { int lo_z, hi_z, lo_y, hi_y, lo_x, hi_x; };

// tensor-map encoding through the runtime's driver entry point (no -lcuda needed); rank 4 or 5, fp32, dense
// last_stride_elems != 0: element stride of the LAST dimension (batch items not densely packed; multiple of 4)
int encode_f32_tiled(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint32_t* box,
                     uint64_t last_stride_elems = 0);
// fp32 pairs: two values in one 64-bit register pair, so that a kernel can carry two voxels through one code path.
// sm_90 has no packed fp32 FMA: fma2 issues two scalar single-rounding FMAs.  The reference's separately rounded
// products and sums are written as a*b = fma(a, b, -0) and a+b = fma(a, 1, b), identity operands passed as kernel
// parameters (see nrt_interp.cu, resize3d kernels, for why).
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pack2(float a, float b) {
  f32x2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ void unpack2(f32x2 v, float& a, float& b) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}


// multi-channel D = 3 warp through the z-marching ring kernel (nrt_warp_march.cu); *used = false when not covered
int warp3d_march(const float* vol, const float* flow, float* out, int B, const int32_t* shape, int C, int method,
                 int has_fill, float fill, int src_z0, int src_n0, int out_z0, int out_n0, int halo,
                 int32_t* err_flag, int64_t vbs, int64_t fbs, int64_t obs, cudaStream_t st, bool* used);

}  // namespace nrt
