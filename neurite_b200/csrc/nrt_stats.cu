// nrt_stats.cu -- per-item reductions of x [items, n]: population SD, max, max |x|, and min with max.  They serve
// GaussianNoise's scale, the Perlin rescaling, min-max normalisation and the MI bin centres.
//
// One partial kernel accumulates min and max of a block's share of an item; its SD instantiation also adds the fp64
// sums {sum d, sum d^2} with d = x - x[item, 0] (the shift makes the variance of a constant item exactly 0).  A warp
// per item then merges the item's block partials in a fixed order: no atomics, deterministic.  max |x| is
// max(-min, max), exact, so it costs the element loop nothing.
//
// Summation order.  An item is read as quads of four consecutive elements (the last one may be short); thread t of
// block b of an item takes quads b * 256 + t, then every (blocks per item * 256)th quad, adding a quad's elements
// in order.  A quad is one float4 load when the item's row is 16-byte aligned and four scalar loads otherwise, so the
// order, and with it an SD, depends on (items, n) only: not on the card, nor on the address of x.
#include "nrt_common.cuh"

namespace nrt {
namespace {

constexpr int kStatThreads = 256;
// Blocks per item: at least 4096 elements each, at most 1024 over the whole batch (one resident wave of the min /
// max kernel on an H100: 8 blocks on each of 132 SMs).  A function of (items, n) only; measured in DESIGN.md §7.
constexpr int kStatBlockElems = 4096;
constexpr int kStatMaxBlocks = 1024;

inline int stat_blocks(int items, int64_t n) {
  const int64_t b = imin64((n + kStatBlockElems - 1) / kStatBlockElems, kStatMaxBlocks / items);
  return (int)(b < 1 ? 1 : b);
}

struct Stats {
  double s1, s2;          // sum d, sum d^2: SD instantiation only
  float mn, mx;
};

__device__ __forceinline__ Stats stats_empty() { return Stats{0.0, 0.0, INFINITY, -INFINITY}; }

template <bool SD>
__device__ __forceinline__ void stats_add(Stats& a, float v, float shift) {
  a.mn = fminf(a.mn, v);
  a.mx = fmaxf(a.mx, v);
  if (SD) {
    const double d = (double)v - (double)shift;
    a.s1 += d;
    a.s2 = fma(d, d, a.s2);
  }
}

template <bool SD>
__device__ __forceinline__ void stats_merge(Stats& a, const Stats& b) {
  a.mn = fminf(a.mn, b.mn);
  a.mx = fmaxf(a.mx, b.mx);
  if (SD) { a.s1 += b.s1; a.s2 += b.s2; }
}

template <bool SD>
__device__ __forceinline__ void stats_warp_reduce(Stats& a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Stats b;
    b.mn = __shfl_xor_sync(0xffffffffu, a.mn, o);
    b.mx = __shfl_xor_sync(0xffffffffu, a.mx, o);
    if (SD) {
      b.s1 = __shfl_xor_sync(0xffffffffu, a.s1, o);
      b.s2 = __shfl_xor_sync(0xffffffffu, a.s2, o);
    }
    stats_merge<SD>(a, b);
  }
}

// grid (blocks per item, items): partial[item * gridDim.x + block].  Without the fp64 sums the kernel fits 32
// registers, 8 blocks per SM; the SD instantiation is left to the compiler (a 40-register cap spills).
template <bool SD>
__global__ void __launch_bounds__(kStatThreads, SD ? 1 : 8)
    item_stats_partial_kernel(const float* __restrict__ x, int64_t n, Stats* __restrict__ partial) {
  const int nbx = gridDim.x, item = blockIdx.y;
  const float* xi = x + (int64_t)item * n;
  const bool vec = (reinterpret_cast<uintptr_t>(xi) & 15u) == 0;
  const float shift = SD ? __ldg(xi) : 0.f;
  const int64_t nq = n >> 2;                 // whole quads
  Stats a = stats_empty();
  int64_t q = (int64_t)blockIdx.x * kStatThreads + threadIdx.x;
  for (; q < nq; q += (int64_t)nbx * kStatThreads) {
    const float* p = xi + (q << 2);
    const float4 v = vec ? ld_stream_f4(reinterpret_cast<const float4*>(p))
                         : make_float4(ld_stream_f(p), ld_stream_f(p + 1), ld_stream_f(p + 2), ld_stream_f(p + 3));
    stats_add<SD>(a, v.x, shift);
    stats_add<SD>(a, v.y, shift);
    stats_add<SD>(a, v.z, shift);
    stats_add<SD>(a, v.w, shift);
  }
  if (q == nq)                               // the short last quad falls to the thread whose turn it is
    for (int64_t i = q << 2; i < n; ++i) stats_add<SD>(a, ld_stream_f(xi + i), shift);
  stats_warp_reduce<SD>(a);
  __shared__ Stats sh[kStatThreads / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kStatThreads / 32; ++w) stats_merge<SD>(a, sh[w]);
    partial[(int64_t)item * nbx + blockIdx.x] = a;
  }
}

// one warp per item
template <bool SD>
__global__ void item_stats_final_kernel(const Stats* __restrict__ partial, int nbx, int64_t n, int kind,
                                        float* __restrict__ out) {
  const int item = blockIdx.x;
  Stats a = stats_empty();
  for (int b = threadIdx.x; b < nbx; b += 32) stats_merge<SD>(a, partial[(int64_t)item * nbx + b]);
  stats_warp_reduce<SD>(a);
  if (threadIdx.x != 0) return;
  if (SD) {
    const double m = a.s1 / (double)n;
    const double var = a.s2 / (double)n - m * m;
    out[item] = (float)sqrt(var > 0.0 ? var : 0.0);
  } else if (kind == NRT_STAT_MAX) {
    out[item] = a.mx;
  } else if (kind == NRT_STAT_ABSMAX) {
    out[item] = fmaxf(0.f, fmaxf(-a.mn, a.mx));       // 0 for an item of NaNs
  } else {
    out[2 * item] = a.mn;
    out[2 * item + 1] = a.mx;
  }
}

template <bool SD>
int launch_item_stats(const float* x, int items, int64_t n, int kind, float* out, Stats* partial, cudaStream_t st) {
  const int nbx = stat_blocks(items, n);
  item_stats_partial_kernel<SD><<<dim3(nbx, items), kStatThreads, 0, st>>>(x, n, partial);
  if (int rc = check_launch("item_stats_partial_kernel")) return rc;
  item_stats_final_kernel<SD><<<items, 32, 0, st>>>(partial, nbx, n, kind, out);
  return check_launch("item_stats_final_kernel");
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int64_t nrt_item_stats_workspace_bytes(int items, int64_t n) {
  if (items < 1) return 0;
  return (int64_t)items * stat_blocks(items, n) * (int64_t)sizeof(Stats);
}

int nrt_item_stats_f32(const float* x, int items, int64_t n, int kind, float* out, void* workspace,
                       int64_t workspace_bytes, void* stream) {
  NRT_REQUIRE(x && out && workspace, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(items >= 1 && items <= 65535, NRT_E_ARG, "items = %d outside 1..65535", items);
  NRT_REQUIRE(n >= 1, NRT_E_ARG, "statistics of an empty item");
  NRT_REQUIRE(kind >= NRT_STAT_SD && kind <= NRT_STAT_MINMAX, NRT_E_ARG, "kind = %d outside 0..3", kind);
  NRT_REQUIRE(workspace_bytes >= nrt_item_stats_workspace_bytes(items, n), NRT_E_ARG, "workspace too small");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Stats* partial = static_cast<Stats*>(workspace);
  return kind == NRT_STAT_SD ? launch_item_stats<true>(x, items, n, kind, out, partial, st)
                             : launch_item_stats<false>(x, items, n, kind, out, partial, st);
}

}  // extern "C"
