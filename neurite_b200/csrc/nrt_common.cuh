// nrt_common.cuh -- shared host/device helpers for libneurite_b200 (sm_90a: TMA, mbarrier).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <stdarg.h>

#include "../../include/neurite_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "libneurite_b200 needs sm_90a (H100): TMA tensor loads and mbarrier transaction counts"
#endif

namespace nrt {

// ---------------------------------------------------------------------------------------
// host side: status + thread-local error string
// ---------------------------------------------------------------------------------------
int set_error(int status, const char* fmt, ...);
int check_launch(const char* what);
int sm_count();

#define NRT_REQUIRE(cond, status, ...) \
  do { if (!(cond)) return ::nrt::set_error((status), __VA_ARGS__); } while (0)

// tiled backward of the D=3, C=1 warp (defined in nrt_interp.cu next to the forward tile kernel)
int warp3d_bwd_tile(const float* vol, const float* flow, const float* gout, float* gvol, float* gflow, int B,
                    const int32_t* shape, int method, int has_fill, cudaStream_t st, bool* used);

// the only reader of the NRT_* test / comparison switches (README.md): unset or empty gives dflt
inline int env_int(const char* name, int dflt) {
  const char* s = getenv(name);
  return (s && *s) ? atoi(s) : dflt;
}

inline int64_t imin64(int64_t a, int64_t b) { return a < b ? a : b; }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---------------------------------------------------------------------------------------
// device side
// ---------------------------------------------------------------------------------------
#ifdef __CUDACC__

// streaming 128-bit load / store that do not pollute L1 (data touched once)
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float ld_stream_f(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream_f(float* p, float v) {
  asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" :: "l"(p), "f"(v) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Per-axis linear-interpolation setup, exactly the reference's op order (utils.py:139-155):
//   x  = clip(loc, 0, max)                (clipped sample position)
//   i0 = clip(floor(loc), 0, max)         == floor(x) because 0 and max are integers
//   i1 = clip(i0 + 1, 0, max)             == min(i0 + 1, max)
//   w1 = i1 - x   (weight of corner bit 0) ;  w0 = 1 - w1  (weight of corner bit 1)
// every operation is a single fp32 rounding (__f*_rn forbids FMA contraction).
struct Axis {
  int i0, i1;
  float wlo, whi;   // weights of corner bit 0 / bit 1
};
__device__ __forceinline__ Axis axis_linear(float loc, float maxf, int maxi) {
  Axis a;
  const float x = fminf(fmaxf(loc, 0.0f), maxf);
  const float f0 = fminf(fmaxf(floorf(loc), 0.0f), maxf);
  const float f1 = fminf(__fadd_rn(f0, 1.0f), maxf);
  a.i0 = min(max(__float2int_rz(f0), 0), maxi);   // min/max only guard NaN input
  a.i1 = min(max(__float2int_rz(f1), 0), maxi);
  a.wlo = __fsub_rn(f1, x);
  a.whi = __fsub_rn(1.0f, a.wlo);
  return a;
}
// nearest: int32(round_half_even(loc)) THEN clip (utils.py:196-197)
__device__ __forceinline__ int axis_nearest(float loc, int maxi) {
  return min(max(__float2int_rn(loc), 0), maxi);
}
// out = out*(!oob) + oob*fill, both products rounded, then the add (utils.py:212-213)
__device__ __forceinline__ float apply_fill(float v, bool oob, float fill) {
  const float keep = oob ? 0.0f : 1.0f;
  const float o = oob ? 1.0f : 0.0f;
  return __fadd_rn(__fmul_rn(v, keep), __fmul_rn(o, fill));
}

// ---- mbarrier / TMA (cp.async.bulk.tensor) primitives ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// bounded wait: a lost TMA transaction traps instead of hanging the GPU box
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (global_timer_ns() - t0 > 4000000000ull) {      // 4 s: a transaction was lost
      if ((threadIdx.x & 31) == 0)
        printf("nrt: mbarrier timeout (block %d thread %d tag %d parity %u smem offset %u)\n", blockIdx.x, threadIdx.x, tag,
               parity, smem_u32(bar));
#ifdef NRT_DEBUG_NO_TRAP
      return;
#else
      __trap();
#endif
    }
  }
}
__device__ __forceinline__ void tma_load_3d(void* dst, const void* tmap, uint64_t* bar,
                                            int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cta.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      :: "r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const void* tmap, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cta.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :: "r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const void* tmap, uint64_t* bar,
                                            int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cta.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      :: "r"(smem_u32(dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" :: "l"(tmap) : "memory");
}
// 1-D bulk copy global -> shared (no descriptor), completes on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
#endif  // __CUDACC__

}  // namespace nrt
