// nrt_lc3d.cu -- LocallyConnected3D (implementation 1) forward for sm_90a.
// Reference: neurite/tf/layers.py:1126-1197 (local_conv), :1098-1101 (bias, activation).
//
// The layer is a weight STREAM: every output position owns a private F x Cout block
// (cfg 4: 432 x 16 fp32 = 27,648 B; 238,328 positions = 6.59 GB) that is used exactly once
// per forward pass, against a 16.8 MB input that lives in L2.  Arithmetic intensity is
// 0.5*B flop/byte, so the kernel is HBM-bound for any realistic batch and the design goal
// is to keep >= ~40 KB of weight loads in flight per SM.
//
//   lc3d_stream_kernel : persistent CTAs; a producer thread streams whole per-position
//       weight blocks into a shared-memory ring with cp.async.bulk (TMA 1-D bulk copy)
//       completing on mbarriers; 4 consumer warps contract a staged block against the
//       position's input patch (gathered from L2 into registers through a shared index
//       table) and release the slot.  One warp owns one position; lanes own fixed
//       4-wide output-channel quads so no weight is read twice.
//   lc3d_generic_kernel: one thread per (b, p, f) -- any Cout / F, used when the fast
//       path's divisibility requirements do not hold.
#include "nrt_interp.cuh"   // CUtensorMap + encode_f32_tiled

namespace nrt {

struct LcGeo {
  int B;
  int I[3];        // input spatial extent
  int O[3];        // output spatial extent (full layer)
  int K[3];
  int St[3];
  int Cin, Cout, F;
  int feature_order;
  int activation;
  int64_t p0, pn;  // this call's output positions [p0, p0+pn)
  int64_t P;       // O0*O1*O2
  int64_t x_batch; // elements per batch item of x
};

__device__ __forceinline__ float activate(float v, int act) {
  switch (act) {
    case NRT_ACT_RELU: return fmaxf(v, 0.f);
    case NRT_ACT_SIGMOID: return __fdiv_rn(1.f, 1.f + expf(-v));
    case NRT_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

// offset of patch feature j inside the input, relative to the patch origin voxel
__device__ __forceinline__ int feature_offset(const LcGeo& g, int j) {
  int i0, i1, i2, c;
  if (g.feature_order == 0) {            // j = ((i0*k1+i1)*k2+i2)*Cin + c
    c = j % g.Cin; j /= g.Cin;
    i2 = j % g.K[2]; j /= g.K[2];
    i1 = j % g.K[1]; i0 = j / g.K[1];
  } else {                               // j = ((c*k0+i0)*k1+i1)*k2+i2
    i2 = j % g.K[2]; j /= g.K[2];
    i1 = j % g.K[1]; j /= g.K[1];
    i0 = j % g.K[0]; c = j / g.K[0];
  }
  return ((i0 * g.I[1] + i1) * g.I[2] + i2) * g.Cin + c;
}

__device__ __forceinline__ int64_t patch_origin(const LcGeo& g, int64_t p) {
  const int o2 = (int)(p % g.O[2]); p /= g.O[2];
  const int o1 = (int)(p % g.O[1]);
  const int o0 = (int)(p / g.O[1]);
  return (((int64_t)o0 * g.St[0] * g.I[1] + (int64_t)o1 * g.St[1]) * g.I[2] + (int64_t)o2 * g.St[2]) * g.Cin;
}

// ---------------------------------------------------------------------------------------
// streaming kernel.  CQ = Cout/4 (power of two <= 32), BB = batch items per pass.
// ---------------------------------------------------------------------------------------
constexpr int kLcMaxWarps = 7;              // consumer groups (<= ring slots - 1) + 1 producer warp
constexpr int kLcMaxStages = 8;

template <int BB, int WPP>
__global__ void __launch_bounds__((kLcMaxWarps * WPP + 1) * 32, 1)
lc3d_stream_kernel(const float* __restrict__ x, const float* __restrict__ kernel,
                   const float* __restrict__ bias, float* __restrict__ out, LcGeo g, int b_base,
                   int stages, int cq_log2) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int CQ = 1 << cq_log2;
  const uint32_t blk_bytes = (uint32_t)g.F * g.Cout * sizeof(float);
  const uint32_t blk_stride = (blk_bytes + 127u) & ~127u;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)stages * blk_stride);
  uint64_t* empty = full + stages;
  int* s_jmap = reinterpret_cast<int*>(empty + stages);                          // [F]

  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
  const int kLcWarps = ((int)(blockDim.x >> 5) - 1) / WPP;     // consumer groups; each group = WPP warps sharing a position
  for (int j = tid; j < g.F; j += (int)blockDim.x) s_jmap[j] = feature_offset(g, j);
  if (tid == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, WPP); }
    fence_mbar_init();
  }
  __syncthreads();

  // This CTA owns positions n_k = blockIdx.x + k*gridDim.x (k = 0, 1, ...): neighbouring
  // CTAs work on neighbouring patches at the same time, so the input stays hot in L2 while
  // the weight stream as a whole advances contiguously.  Step k uses ring slot k % stages
  // and is consumed by warp k % kLcWarps.
  if (wid == kLcWarps * WPP) {
    // ===== producer: one thread streams weight blocks into the ring =====
    if (lane == 0) {
      int k = 0;
      for (int64_t n = blockIdx.x; n < g.pn; n += gridDim.x, ++k) {
        const int slot = k % stages;
        const int round = k / stages;
        if (round >= 1) mbar_wait(empty + slot, (uint32_t)((round - 1) & 1));   // slot released
        mbar_expect_tx(full + slot, blk_bytes);
        bulk_load_1d(smem_raw + (size_t)slot * blk_stride, kernel + n * (int64_t)g.F * g.Cout,
                     blk_bytes, full + slot);
      }
    }
    return;
  }

  // ===== consumer warps =====
  // One warp per position.  Lane l reads float4 l, l+32, ... of the staged weight block:
  // patch feature j = i / CQ, output-channel quad fq = i % CQ = l % CQ (fixed per lane), so the
  // block is read exactly once, conflict-free, and each lane keeps BB x 4 accumulators.
  const int n4 = g.F * CQ;                      // float4s per block
  const int fq = lane & (CQ - 1);
  // The input values a lane needs do not depend on the weights: gather a chunk of them from
  // L1/L2 into registers first (CH*BB independent loads in flight; the first chunk is issued
  // before waiting for the TMA), then run the LDS.128 + FFMA chain with no global latency in it.
  constexpr int CH = (27 * BB <= 54) ? 27 : (48 / BB);
  const int iters = (n4 + 31) >> 5;
  // WPP warps share a position: warp `sub` of the group contracts batch items
  // [b_base + sub*BB, b_base + (sub+1)*BB) against the same staged weight block.
  const int grp = wid / WPP, sub = wid - grp * WPP;
  const int b0 = b_base + sub * BB;
  int k = grp;
  for (int64_t n = (int64_t)blockIdx.x + (int64_t)grp * gridDim.x; n < g.pn;
       n += (int64_t)kLcWarps * gridDim.x, k += kLcWarps) {
    const int slot = k % stages;
    const uint32_t ph = (uint32_t)((k / stages) & 1);
    const float* xp = x + (int64_t)b0 * g.x_batch + patch_origin(g, g.p0 + n);
    float acc[BB][4];
#pragma unroll
    for (int b = 0; b < BB; ++b) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.f;
    const float4* w4 = reinterpret_cast<const float4*>(smem_raw + (size_t)slot * blk_stride);
    for (int i0 = 0; i0 < iters; i0 += CH) {
      float xv[CH][BB];
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int i = lane + ((i0 + c) << 5);
        const int off = (i < n4) ? s_jmap[i >> cq_log2] : 0;
#pragma unroll
        for (int b = 0; b < BB; ++b) xv[c][b] = __ldg(xp + (int64_t)b * g.x_batch + off);
      }
      if (i0 == 0) {
        // parity aliasing guard (see lc3d_patch_kernel): the previous round of this slot must have been consumed
        if (k >= stages) mbar_wait(empty + slot, ph ^ 1u);
        mbar_wait(full + slot, ph);
      }
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int i = lane + ((i0 + c) << 5);
        // past the end of the block the weights are zero (no branch: the accumulators stay in place)
        const float4 wv = (i < n4) ? w4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int b = 0; b < BB; ++b) {
          acc[b][0] = fmaf(xv[c][b], wv.x, acc[b][0]);
          acc[b][1] = fmaf(xv[c][b], wv.y, acc[b][1]);
          acc[b][2] = fmaf(xv[c][b], wv.z, acc[b][2]);
          acc[b][3] = fmaf(xv[c][b], wv.w, acc[b][3]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) {                             // slot free: every lane has read its share
      asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(empty + slot)) : "memory");
    }
    // fold the 32/CQ lanes that share an output quad
#pragma unroll
    for (int b = 0; b < BB; ++b)
#pragma unroll
      for (int q = 0; q < 4; ++q)
        for (int o = 16; o >= CQ; o >>= 1) acc[b][q] += __shfl_xor_sync(0xffffffffu, acc[b][q], o);
    if (lane < CQ) {
      float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (bias) bv = __ldg(reinterpret_cast<const float4*>(bias + n * g.Cout) + fq);
#pragma unroll
      for (int b = 0; b < BB; ++b) {
        float4 r;
        r.x = activate(acc[b][0] + bv.x, g.activation);
        r.y = activate(acc[b][1] + bv.y, g.activation);
        r.z = activate(acc[b][2] + bv.z, g.activation);
        r.w = activate(acc[b][3] + bv.w, g.activation);
        reinterpret_cast<float4*>(out + ((int64_t)(b0 + b) * g.pn + n) * g.Cout)[fq] = r;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// patch kernel (batch > 1).  lc3d_stream_kernel gathers a position's input patch lane by lane from L2: at
// batch 8 that is 216 scalar loads per lane and ~6 integer instructions of addressing each -- ~7100 warp
// instructions per position, which keeps the ALU pipe busy instead of the weight stream.
// Here the producer thread fetches the patch with ONE TMA tensor load per position -- the box
// (Cin, K2, K1, K0, NB) of the channels-last input [B, I0, I1, I2, Cin] lands in shared memory as [b][j] with
// exactly the reference's feature order j = ((i0*K1 + i1)*K2 + i2)*Cin + c (layers.py:1173-1188) -- on the same
// mbarrier as the weight block, and a lane reads its input values with conflict-free broadcast LDS.
// ---------------------------------------------------------------------------------------
template <int BB, int WPP>
__global__ void __launch_bounds__((kLcMaxWarps * WPP + 1) * 32, 1)
lc3d_patch_kernel(const __grid_constant__ CUtensorMap tm_x, const float* __restrict__ kernel,
                  const float* __restrict__ bias, float* __restrict__ out, LcGeo g, int b_base,
                  int stages, int cq_log2) {
  constexpr int NB = BB * WPP;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int CQ = 1 << cq_log2;
  const uint32_t blk_bytes = (uint32_t)g.F * g.Cout * sizeof(float);
  const uint32_t patch_bytes = (uint32_t)g.F * NB * sizeof(float);
  const uint32_t patch_off = (blk_bytes + 127u) & ~127u;
  const uint32_t slot_stride = (patch_off + patch_bytes + 127u) & ~127u;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)stages * slot_stride);
  uint64_t* empty = full + stages;
  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
  const int groups = ((int)(blockDim.x >> 5) - 1) / WPP;
  if (tid == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, WPP); }
    fence_mbar_init();
  }
  __syncthreads();
  if (wid == groups * WPP) {
    if (lane == 0) {
      int k = 0;
      for (int64_t n = blockIdx.x; n < g.pn; n += gridDim.x, ++k) {
        const int slot = k % stages, round = k / stages;
        if (round >= 1) mbar_wait(empty + slot, (uint32_t)((round - 1) & 1), 1000000 + k);
        unsigned char* dst = smem_raw + (size_t)slot * slot_stride;
        mbar_expect_tx(full + slot, blk_bytes + patch_bytes);
        bulk_load_1d(dst, kernel + n * (int64_t)g.F * g.Cout, blk_bytes, full + slot);
        int64_t p = g.p0 + n;
        const int o2 = (int)(p % g.O[2]); p /= g.O[2];
        const int o1 = (int)(p % g.O[1]);
        const int o0 = (int)(p / g.O[1]);
        tma_load_5d(dst + patch_off, &tm_x, full + slot, 0, o2 * g.St[2], o1 * g.St[1], o0 * g.St[0], b_base);
      }
    }
    return;
  }
  const int n4 = g.F * CQ;                      // float4s per weight block
  const int fq = lane & (CQ - 1);
  const int grp = wid / WPP, sub = wid - grp * WPP;
  const int b0 = b_base + sub * BB;
  int k = grp;
  for (int64_t n = (int64_t)blockIdx.x + (int64_t)grp * gridDim.x; n < g.pn; n += (int64_t)groups * gridDim.x, k += groups) {
    const int slot = k % stages;
    const uint32_t ph = (uint32_t)((k / stages) & 1);
    const unsigned char* base = smem_raw + (size_t)slot * slot_stride;
    const float4* w4 = reinterpret_cast<const float4*>(base);
    const float* sx = reinterpret_cast<const float*>(base + patch_off) + (size_t)sub * BB * g.F;
    float acc[BB][4];
#pragma unroll
    for (int b = 0; b < BB; ++b) acc[b][0] = acc[b][1] = acc[b][2] = acc[b][3] = 0.f;
    // Parity aliasing guard.  A group visits only every `groups`-th step, so it may reach for step k while the PREVIOUS
    // use of this slot (step k - stages, another group's) is still in flight: copies of different steps can complete
    // out of order (the patch comes through the tensor path, the weights through the bulk path), the barrier would
    // still be one phase behind and try_wait on the next parity would return at once -- on a half-filled slot.
    // First make sure the previous round of the slot has been CONSUMED (which implies it had landed); the `empty`
    // barrier cannot be more than one phase away from what this warp expects, so that wait cannot alias.
    // (Seen as a 4 s mbarrier timeout at full size, batch 2 -- never with the sanitizer's slower timing.)
    if (k >= stages) mbar_wait(empty + slot, ph ^ 1u, 2000000 + k);
    mbar_wait(full + slot, ph, k);
    // lane l reads float4 l, l+32, ... of the weight block: patch feature j = i / CQ advances by 32 / CQ per step
    const float4* wp = w4 + lane;
    const float* xp = sx + (lane >> cq_log2);
    const int xstep = 32 >> cq_log2;
#define NRT_LC_STEP(WV, XP)                                                                              \
    do {                                                                                                 \
      _Pragma("unroll") for (int b = 0; b < BB; ++b) {                                                   \
        const float xv = (XP)[b * g.F];                                                                  \
        acc[b][0] = fmaf(xv, (WV).x, acc[b][0]);                                                         \
        acc[b][1] = fmaf(xv, (WV).y, acc[b][1]);                                                         \
        acc[b][2] = fmaf(xv, (WV).z, acc[b][2]);                                                         \
        acc[b][3] = fmaf(xv, (WV).w, acc[b][3]);                                                         \
      }                                                                                                  \
    } while (0)
    const int full_iters = n4 >> 5;
#pragma unroll 6
    for (int c = 0; c < full_iters; ++c, wp += 32, xp += xstep) {
      const float4 wv = *wp;
      NRT_LC_STEP(wv, xp);
    }
    if ((n4 & 31) && lane + (full_iters << 5) < n4) {            // ragged tail of the block
      const float4 wv = *wp;
      NRT_LC_STEP(wv, xp);
    }
#undef NRT_LC_STEP
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + slot);      // slot free: every lane has read its share
    // fold the 32/CQ lanes that share an output quad
#pragma unroll
    for (int b = 0; b < BB; ++b)
#pragma unroll
      for (int q = 0; q < 4; ++q)
        for (int o = 16; o >= CQ; o >>= 1) acc[b][q] += __shfl_xor_sync(0xffffffffu, acc[b][q], o);
    if (lane < CQ) {
      float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (bias) bv = __ldg(reinterpret_cast<const float4*>(bias + n * g.Cout) + fq);
#pragma unroll
      for (int b = 0; b < BB; ++b) {
        float4 r;
        r.x = activate(acc[b][0] + bv.x, g.activation);
        r.y = activate(acc[b][1] + bv.y, g.activation);
        r.z = activate(acc[b][2] + bv.z, g.activation);
        r.w = activate(acc[b][3] + bv.w, g.activation);
        reinterpret_cast<float4*>(out + ((int64_t)(b0 + b) * g.pn + n) * g.Cout)[fq] = r;
      }
    }
  }
}


// ---------------------------------------------------------------------------------------
// row kernel (batch >= 4, Cout = 16).  In lc3d_patch_kernel a lane owns ONE output quad and a slice of the patch
// features: per float4 of weights it gets from shared memory (16 B) and per input value (4 B) it issues 4 * BB FMAs,
// i.e. 2-3 bytes of shared-memory traffic per FMA and lane.  The shared-memory crossbar delivers 128 B per clock and SM,
// the FMA pipes take 128 lane-FMAs per clock, so at batch 8 that kernel is bound by the crossbar, not by the weight
// stream from HBM.
// Here a lane owns patch ROWS j = lane, lane + 32, ... and ALL 16 output channels of BB batch items: a weight row
// (64 B) and BB input values feed 16 * BB FMAs -- 0.6-0.75 B per FMA and lane -- and the 16 * BB partial sums of the
// 32 lanes are folded once per position with a reduce-scatter of shuffles (each step halves what a lane still holds).
// Bank conflicts: rows are 64 B apart, so the lanes of a quarter-warp would hit two bank groups with the same chunk of
// their rows; lane l therefore reads its row's four 16-byte chunks in the order q ^ m, m = (l >> 1) & 3, and accumulates
// chunk q ^ m in register set q.
// The fold needs no selects.  Final owner of (item, chunk): item from lane bits 4, 3 (and 0 at eight items), chunk
// from lane bits 2, 1 -- i.e. chunk m.  (a) A lane keeps batch SLOT b for item b ^ pb, pb = its own item: its lower
// slots then hold the items it must keep at every batch step (mask 16, 8, 1: partners that share m) and it hands over
// the upper half.  (b) Register set 0 holds chunk 0 ^ m = the lane's own chunk, and set d holds chunk m ^ d = the own
// chunk of lane l ^ 2d: one shuffle per set and value sends every chunk to its owner.
// Same ring, barriers and TMA patch load as lc3d_patch_kernel.  Summation order differs from the other kernels
// (rows are summed lane-wise first): results agree to fp32 rounding, not bit for bit.
// Batch 4 keeps lc3d_patch_kernel<2,2>; batch 8 and more take <4,2> (two warps x four items per position).
// ---------------------------------------------------------------------------------------
template <int N>
__device__ __forceinline__ void fold_upper(float* v, int mask) {      // v[0 .. N/2) += partner's v[N/2 .. N)
#pragma unroll
  for (int i = 0; i < N / 2; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i + N / 2], mask);
}

template <int BB, int WPP>
__global__ void __launch_bounds__((kLcMaxWarps * WPP + 1) * 32, 1)
lc3d_rows_kernel(const __grid_constant__ CUtensorMap tm_x, const float* __restrict__ kernel,
                 const float* __restrict__ bias, float* __restrict__ out, LcGeo g, int b_base, int stages) {
  static_assert(BB == 4 || BB == 8, "the fold is written for 4 or 8 batch items per warp (8: measured slower, not built)");
  constexpr int NB = BB * WPP;
  constexpr int CO = 16;                                 // output channels (host checks g.Cout == 16)
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t blk_bytes = (uint32_t)g.F * CO * sizeof(float);
  const uint32_t patch_bytes = (uint32_t)g.F * NB * sizeof(float);
  const uint32_t patch_off = (blk_bytes + 127u) & ~127u;
  const uint32_t slot_stride = (patch_off + patch_bytes + 127u) & ~127u;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)stages * slot_stride);
  uint64_t* empty = full + stages;
  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
  const int groups = ((int)(blockDim.x >> 5) - 1) / WPP;
  if (tid == 0) {
    for (int s = 0; s < stages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, WPP); }
    fence_mbar_init();
  }
  __syncthreads();
  if (wid == groups * WPP) {                             // producer: identical to lc3d_patch_kernel's
    if (lane == 0) {
      int k = 0;
      for (int64_t n = blockIdx.x; n < g.pn; n += gridDim.x, ++k) {
        const int slot = k % stages, round = k / stages;
        if (round >= 1) mbar_wait(empty + slot, (uint32_t)((round - 1) & 1), 1000000 + k);
        unsigned char* dst = smem_raw + (size_t)slot * slot_stride;
        mbar_expect_tx(full + slot, blk_bytes + patch_bytes);
        bulk_load_1d(dst, kernel + n * (int64_t)g.F * CO, blk_bytes, full + slot);
        int64_t p = g.p0 + n;
        const int o2 = (int)(p % g.O[2]); p /= g.O[2];
        const int o1 = (int)(p % g.O[1]);
        const int o0 = (int)(p / g.O[1]);
        tma_load_5d(dst + patch_off, &tm_x, full + slot, 0, o2 * g.St[2], o1 * g.St[1], o0 * g.St[0], b_base);
      }
    }
    return;
  }
  const int grp = wid / WPP, sub = wid - grp * WPP;
  const int b0 = b_base + sub * BB;
  const int m = (lane >> 1) & 3;                         // chunk permutation of this lane = the chunk it ends up with
  // the item this lane ends up with; batch slot b of the lane accumulates item b ^ pb
  const int pb = BB == 8 ? ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + (lane & 1) : ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);
  int xoff[BB];
#pragma unroll
  for (int b = 0; b < BB; ++b) xoff[b] = (b ^ pb) * g.F;
  const int iters = (g.F + 31) >> 5;
  int k = grp;
  for (int64_t n = (int64_t)blockIdx.x + (int64_t)grp * gridDim.x; n < g.pn; n += (int64_t)groups * gridDim.x, k += groups) {
    const int slot = k % stages;
    const uint32_t ph = (uint32_t)((k / stages) & 1);
    const unsigned char* base = smem_raw + (size_t)slot * slot_stride;
    // this lane's first row, its four chunks in the lane's order; a row step of 32 is 512 float4
    const float4* wq0 = reinterpret_cast<const float4*>(base) + lane * 4 + (0 ^ m);
    const float4* wq1 = reinterpret_cast<const float4*>(base) + lane * 4 + (1 ^ m);
    const float4* wq2 = reinterpret_cast<const float4*>(base) + lane * 4 + (2 ^ m);
    const float4* wq3 = reinterpret_cast<const float4*>(base) + lane * 4 + (3 ^ m);
    const float* xp = reinterpret_cast<const float*>(base + patch_off) + (size_t)sub * BB * g.F + lane;
    float v[BB * 16];                                    // [slot][register set q][e] = channel 4 * (q ^ m) + e
#pragma unroll
    for (int i = 0; i < BB * 16; ++i) v[i] = 0.f;
    if (k >= stages) mbar_wait(empty + slot, ph ^ 1u, 2000000 + k);      // parity aliasing guard (lc3d_patch_kernel)
    mbar_wait(full + slot, ph, k);
#pragma unroll 2
    for (int c = 0; c < iters; ++c) {
      if (lane + (c << 5) < g.F) {                       // ragged last step: rows past F do not exist
        const float4 w0 = wq0[c * 128], w1 = wq1[c * 128], w2 = wq2[c * 128], w3 = wq3[c * 128];
        const float w[16] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w,
                             w2.x, w2.y, w2.z, w2.w, w3.x, w3.y, w3.z, w3.w};
#pragma unroll
        for (int b = 0; b < BB; ++b) {
          const float xv = xp[xoff[b] + (c << 5)];
#pragma unroll
          for (int i = 0; i < 16; ++i) v[b * 16 + i] = fmaf(xv, w[i], v[b * 16 + i]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + slot);            // slot free: every lane has read its rows
    // ---- fold the 32 lanes' partial sums: v[slot][register set][channel in chunk]
    fold_upper<BB * 16>(v, 16);
    fold_upper<BB * 8>(v, 8);
    if (BB == 8) fold_upper<BB * 4>(v, 1);
    // slot 0 = item pb, 16 values [set][e]; every other set goes to the lane that owns its chunk
    float u[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      u[e] = v[e] + __shfl_xor_sync(0xffffffffu, v[4 + e], 2);
      u[e] += __shfl_xor_sync(0xffffffffu, v[8 + e], 4);
      u[e] += __shfl_xor_sync(0xffffffffu, v[12 + e], 6);
    }
    if (BB == 4) {                                       // lanes l and l ^ 1 hold two halves of the same sum
#pragma unroll
      for (int e = 0; e < 4; ++e) u[e] += __shfl_xor_sync(0xffffffffu, u[e], 1);
    }
    if (BB == 8 || (lane & 1) == 0) {
      const int ch = m * 4;
      const float4 bv = bias ? __ldg(reinterpret_cast<const float4*>(bias + n * CO + ch)) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 r;
      r.x = activate(u[0] + bv.x, g.activation); r.y = activate(u[1] + bv.y, g.activation);
      r.z = activate(u[2] + bv.z, g.activation); r.w = activate(u[3] + bv.w, g.activation);
      *reinterpret_cast<float4*>(out + ((int64_t)(b0 + pb) * g.pn + n) * CO + ch) = r;
    }
  }
}

// ---------------------------------------------------------------------------------------
// generic kernel: one thread per (b, position, filter)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
lc3d_generic_kernel(const float* __restrict__ x, const float* __restrict__ kernel,
                    const float* __restrict__ bias, float* __restrict__ out, LcGeo g) {
  const int64_t total = (int64_t)g.B * g.pn * g.Cout;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int f = (int)(t % g.Cout);
    const int64_t n = (t / g.Cout) % g.pn;
    const int b = (int)(t / ((int64_t)g.Cout * g.pn));
    const float* xp = x + (int64_t)b * g.x_batch + patch_origin(g, g.p0 + n);
    const float* wp = kernel + n * (int64_t)g.F * g.Cout + f;
    float acc = 0.f;
    for (int j = 0; j < g.F; ++j) acc = fmaf(__ldg(xp + feature_offset(g, j)), __ldg(wp + (int64_t)j * g.Cout), acc);
    if (bias) acc += __ldg(bias + n * g.Cout + f);
    out[t] = activate(acc, g.activation);
  }
}

// ---------------------------------------------------------------------------------------
// backward: one warp per output position, lanes own fixed output-channel quads like the
// forward.  In one pass over the position's weight block:
//   grad_kernel[p,j,f] = sum_b patch[b,p,j] * dy[b,p,f]          (6.59 GB write stream at cfg 4)
//   grad_x[b, patch(p,j)] += sum_f dy[b,p,f] * kernel[p,j,f]     (scatter: patches overlap -> atomics)
// grad_bias[p,f] = sum_b dy[b,p,f] is a plain reduction done by the caller.
// ---------------------------------------------------------------------------------------
template <int BB>
__global__ void __launch_bounds__(256)
lc3d_bwd_kernel(const float* __restrict__ x, const float* __restrict__ kernel, const float* __restrict__ dy,
                float* __restrict__ gx, float* __restrict__ gk, LcGeo g, int b_base, int cq_log2, int accumulate_gk) {
  extern __shared__ int s_jmap[];
  const int CQ = 1 << cq_log2;
  for (int j = threadIdx.x; j < g.F; j += blockDim.x) s_jmap[j] = feature_offset(g, j);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int fq = lane & (CQ - 1);
  const int n4 = g.F * CQ;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); n < g.pn; n += warps) {
    const int64_t po = patch_origin(g, g.p0 + n);
    float4 d4[BB];
#pragma unroll
    for (int b = 0; b < BB; ++b)
      d4[b] = __ldg(reinterpret_cast<const float4*>(dy + ((int64_t)(b_base + b) * g.pn + n) * g.Cout) + fq);
    const float4* w4 = reinterpret_cast<const float4*>(kernel + n * (int64_t)g.F * g.Cout);
    float4* gk4 = gk ? reinterpret_cast<float4*>(gk + n * (int64_t)g.F * g.Cout) : nullptr;
    for (int i0 = 0; i0 < n4; i0 += 32) {              // warp-uniform trip count (shuffles inside)
      const int i = i0 + lane;
      const bool valid = i < n4;
      const int off = valid ? s_jmap[i >> cq_log2] : 0;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gx && valid) wv = ld_stream_f4(w4 + i);
#pragma unroll
      for (int b = 0; b < BB; ++b) {
        if (gk && valid) {
          const float xv = __ldg(x + (int64_t)(b_base + b) * g.x_batch + po + off);
          acc.x = fmaf(xv, d4[b].x, acc.x); acc.y = fmaf(xv, d4[b].y, acc.y);
          acc.z = fmaf(xv, d4[b].z, acc.z); acc.w = fmaf(xv, d4[b].w, acc.w);
        }
        if (gx) {
          float part = (wv.x * d4[b].x + wv.y * d4[b].y) + (wv.z * d4[b].z + wv.w * d4[b].w);
          for (int o = CQ >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
          if (fq == 0 && valid) atomicAdd(gx + (int64_t)(b_base + b) * g.x_batch + po + off, part);
        }
      }
      if (gk && valid) {
        if (accumulate_gk) {
          const float4 old = gk4[i];
          acc.x += old.x; acc.y += old.y; acc.z += old.z; acc.w += old.w;
        }
        st_stream_f4(gk4 + i, acc);
      }
    }
  }
}

template <int BB, int WPP>
static int launch_stream(const float* x, const float* kernel, const float* bias, float* out, const LcGeo& g,
                         int b_base, int cq_log2, cudaStream_t st) {
  const uint32_t blk_bytes = (uint32_t)g.F * g.Cout * sizeof(float);
  const uint32_t blk_stride = (blk_bytes + 127u) & ~127u;
  const size_t fixed = (size_t)g.F * sizeof(int) + 2 * kLcMaxStages * sizeof(uint64_t) + 128;
  int stages = (int)((220 * 1024 - fixed) / (size_t)blk_stride);
  if (stages < 2) return 1;                      // caller falls back to the generic kernel
  if (stages > kLcMaxStages) stages = kLcMaxStages;
  const size_t smem = (size_t)stages * blk_stride + (size_t)stages * 16 + (size_t)g.F * sizeof(int) + 16;
  auto kern = lc3d_stream_kernel<BB, WPP>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("cudaFuncSetAttribute(lc3d_stream)");
  int grid = sm_count();
  if (g.pn < grid) grid = (int)g.pn;
  int nw = env_int("NRT_LC3D_WARPS", kLcMaxWarps);   // as many consumer groups as the ring allows (measured best)
  if (nw < 1) nw = 1;
  if (nw > kLcMaxWarps) nw = kLcMaxWarps;
  if (nw > stages - 1) nw = stages - 1;
  kern<<<grid, (nw * WPP + 1) * 32, smem, st>>>(x, kernel, bias, out, g, b_base, stages, cq_log2);
  return check_launch("lc3d_stream_kernel");
}

// batch > 1: weights by bulk copy + the position's input patch by one TMA tensor load (lc3d_patch_kernel).
// Returns 1 when the geometry is not covered (caller takes lc3d_stream_kernel).
template <int BB, int WPP>
static int launch_patch(const float* x, const float* kernel, const float* bias, float* out, const LcGeo& g,
                        int b_base, int cq_log2, cudaStream_t st) {
  constexpr int NB = BB * WPP;
  if (g.feature_order != 0 || g.Cin % 4 != 0 || g.Cin > 256 || g.K[0] > 256 || g.K[1] > 256 || g.K[2] > 256 || !aligned16(x))
    return 1;
  const uint32_t blk_bytes = (uint32_t)g.F * g.Cout * sizeof(float);
  const uint32_t patch_bytes = (uint32_t)g.F * NB * sizeof(float);
  const uint32_t patch_off = (blk_bytes + 127u) & ~127u;
  const uint32_t slot_stride = (patch_off + patch_bytes + 127u) & ~127u;
  int stages = (int)((220 * 1024 - 2 * kLcMaxStages * sizeof(uint64_t) - 128) / (size_t)slot_stride);
  if (stages < 3) return 1;
  if (stages > kLcMaxStages) stages = kLcMaxStages;
  const int forced_stages = env_int("NRT_LC3D_STAGES", 0);
  if (forced_stages >= 3 && forced_stages < stages) stages = forced_stages;
  const size_t smem = (size_t)stages * slot_stride + (size_t)stages * 16 + 16;
  CUtensorMap tmx;
  const uint64_t xd[5] = {(uint64_t)g.Cin, (uint64_t)g.I[2], (uint64_t)g.I[1], (uint64_t)g.I[0], (uint64_t)g.B};
  const uint32_t xb[5] = {(uint32_t)g.Cin, (uint32_t)g.K[2], (uint32_t)g.K[1], (uint32_t)g.K[0], (uint32_t)NB};
  int rc = encode_f32_tiled(&tmx, x, 5, xd, xb);
  if (rc != NRT_OK) return rc;
  auto kern = lc3d_patch_kernel<BB, WPP>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("cudaFuncSetAttribute(lc3d_patch)");
  int grid = sm_count();
  if (g.pn < grid) grid = (int)g.pn;
  int nw = env_int("NRT_LC3D_WARPS", kLcMaxWarps);
  if (nw < 1) nw = 1;
  if (nw > kLcMaxWarps) nw = kLcMaxWarps;
  if (nw > stages - 1) nw = stages - 1;
  kern<<<grid, (nw * WPP + 1) * 32, smem, st>>>(tmx, kernel, bias, out, g, b_base, stages, cq_log2);
  return check_launch("lc3d_patch_kernel");
}

// batch >= 4 with 16 output channels: rows owned by lanes, all channels per lane (lc3d_rows_kernel).
// Returns 1 when the geometry is not covered (caller takes lc3d_patch_kernel).
template <int BB, int WPP>
static int launch_rows(const float* x, const float* kernel, const float* bias, float* out, const LcGeo& g,
                       int b_base, cudaStream_t st) {
  constexpr int NB = BB * WPP;
  if (g.Cout != 16 || g.feature_order != 0 || g.Cin % 4 != 0 || g.Cin > 256 || g.K[0] > 256 || g.K[1] > 256 ||
      g.K[2] > 256 || !aligned16(x) || (bias && (reinterpret_cast<uintptr_t>(bias) & 15u) != 0))
    return 1;
  const uint32_t blk_bytes = (uint32_t)g.F * 16 * sizeof(float);
  const uint32_t patch_bytes = (uint32_t)g.F * NB * sizeof(float);
  const uint32_t patch_off = (blk_bytes + 127u) & ~127u;
  const uint32_t slot_stride = (patch_off + patch_bytes + 127u) & ~127u;
  int stages = (int)((220 * 1024 - 2 * kLcMaxStages * sizeof(uint64_t) - 128) / (size_t)slot_stride);
  if (stages < 3) return 1;
  if (stages > kLcMaxStages) stages = kLcMaxStages;
  const int forced_stages = env_int("NRT_LC3D_STAGES", 0);
  if (forced_stages >= 3 && forced_stages < stages) stages = forced_stages;
  const size_t smem = (size_t)stages * slot_stride + (size_t)stages * 16 + 16;
  CUtensorMap tmx;
  const uint64_t xd[5] = {(uint64_t)g.Cin, (uint64_t)g.I[2], (uint64_t)g.I[1], (uint64_t)g.I[0], (uint64_t)g.B};
  const uint32_t xb[5] = {(uint32_t)g.Cin, (uint32_t)g.K[2], (uint32_t)g.K[1], (uint32_t)g.K[0], (uint32_t)NB};
  int rc = encode_f32_tiled(&tmx, x, 5, xd, xb);
  if (rc != NRT_OK) return rc;
  auto kern = lc3d_rows_kernel<BB, WPP>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return check_launch("cudaFuncSetAttribute(lc3d_rows)");
  int grid = sm_count();
  if (g.pn < grid) grid = (int)g.pn;
  int nw = env_int("NRT_LC3D_WARPS", kLcMaxWarps);   // consumer groups: as many as the ring allows, one slot left in flight
  if (nw < 1) nw = 1;
  if (nw > kLcMaxWarps) nw = kLcMaxWarps;
  if (nw > stages - 1) nw = stages - 1;
  kern<<<grid, (nw * WPP + 1) * 32, smem, st>>>(tmx, kernel, bias, out, g, b_base, stages);
  return check_launch("lc3d_rows_kernel");
}

}  // namespace nrt

using namespace nrt;

extern "C" int nrt_lc3d_fwd_f32(const float* x, const float* kernel, const float* bias, float* out, int B,
                                const int32_t* in_shape, int Cin, int Cout, const int32_t* ksize,
                                const int32_t* strides, int feature_order, int activation, int64_t p0,
                                int64_t p_count, void* stream) {
  NRT_REQUIRE(x && kernel && out && in_shape && ksize && strides, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1, NRT_E_ARG, "bad B/Cin/Cout");
  NRT_REQUIRE(feature_order == 0 || feature_order == 1, NRT_E_ARG, "feature_order must be 0 or 1");
  NRT_REQUIRE(activation >= NRT_ACT_LINEAR && activation <= NRT_ACT_TANH, NRT_E_ARG, "unknown activation %d", activation);
  LcGeo g;
  g.B = B; g.Cin = Cin; g.Cout = Cout; g.feature_order = feature_order; g.activation = activation;
  g.P = 1; g.x_batch = Cin;
  int64_t F = Cin;
  for (int d = 0; d < 3; ++d) {
    g.I[d] = in_shape[d]; g.K[d] = ksize[d]; g.St[d] = strides[d];
    NRT_REQUIRE(g.I[d] >= 1 && g.K[d] >= 1 && g.St[d] >= 1 && g.K[d] <= g.I[d], NRT_E_ARG,
                "bad input/kernel/stride at axis %d", d);
    g.O[d] = (g.I[d] - g.K[d]) / g.St[d] + 1;            // conv_output_length, 'valid'
    g.P *= g.O[d]; g.x_batch *= g.I[d]; F *= g.K[d];
  }
  NRT_REQUIRE(F <= 1 << 20 && g.x_batch <= 0x7fffffffLL, NRT_E_SIZE, "patch or input too large");
  g.F = (int)F;
  NRT_REQUIRE(p0 >= 0 && p_count >= 0 && p0 + p_count <= g.P, NRT_E_ARG,
              "positions [%lld,%lld) outside [0,%lld)", (long long)p0, (long long)(p0 + p_count), (long long)g.P);
  g.p0 = p0; g.pn = p_count;
  if (B == 0 || p_count == 0) return NRT_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  const int cq = Cout / 4;
  const bool fast = (Cout % 4 == 0) && cq <= 32 && (cq & (cq - 1)) == 0 && aligned16(kernel) && aligned16(out) &&
                    (!bias || aligned16(bias)) && ((int64_t)g.F * Cout * 4) % 16 == 0 && g.F <= 8192 &&
                    env_int("NRT_LC3D_GENERIC", 0) == 0;
  if (fast) {
    int cq_log2 = 0;
    while ((1 << cq_log2) < cq) ++cq_log2;
    int b = 0, rc = NRT_OK;
    const bool patch = env_int("NRT_LC3D_PATCH", 1) != 0;
    while (b < B && rc == NRT_OK) {              // batch items per pass = BB * WPP (weights streamed once per pass)
      const int left = B - b;
      // one batch item: the TMA-patch kernel too
      if (patch && left == 1 && env_int("NRT_LC3D_PATCH1", 1)) {
        const int prc = launch_patch<1, 1>(x, kernel, bias, out, g, b, cq_log2, st);
        if (prc <= 0) { rc = prc; b += 1; continue; }
      }
      if (patch && left >= 2) {
        // batch > 1: the position's input patch arrives by TMA next to its weight block (lc3d_patch_kernel)
        int prc;
        if (left >= 8) {
          // row kernel (lanes own patch rows and all 16 channels; two warps x four items per position), else -- other
          // channel counts, NRT_LC3D_ROWS=0 -- the patch kernel (lanes own an output quad; four warps x two items)
          prc = env_int("NRT_LC3D_ROWS", 1) ? launch_rows<4, 2>(x, kernel, bias, out, g, b, st) : 1;
          if (prc == 1) prc = launch_patch<2, 4>(x, kernel, bias, out, g, b, cq_log2, st);
          if (prc <= 0) { rc = prc; b += 8; continue; }
        }
        else if (left >= 4) { prc = launch_patch<2, 2>(x, kernel, bias, out, g, b, cq_log2, st); if (prc <= 0) { rc = prc; b += 4; continue; } }
        else {
          // two batch items: two warps per position, one item each (one warp doing both measured slower)
          prc = launch_patch<1, 2>(x, kernel, bias, out, g, b, cq_log2, st);
          if (prc <= 0) { rc = prc; b += 2; continue; }
        }
      }
      if (left >= 8) { rc = launch_stream<4, 2>(x, kernel, bias, out, g, b, cq_log2, st); b += 8; }
      else if (left >= 4) { rc = launch_stream<2, 2>(x, kernel, bias, out, g, b, cq_log2, st); b += 4; }
      else if (left >= 2) { rc = launch_stream<2, 1>(x, kernel, bias, out, g, b, cq_log2, st); b += 2; }
      else { rc = launch_stream<1, 1>(x, kernel, bias, out, g, b, cq_log2, st); b += 1; }
    }
    if (rc <= 0) return rc;       // rc == 1: weight block does not fit the ring -> generic
  }
  const int64_t total = (int64_t)B * g.pn * Cout;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 32);
  lc3d_generic_kernel<<<grid, 256, 0, st>>>(x, kernel, bias, out, g);
  return check_launch("lc3d_generic_kernel");
}

extern "C" int nrt_lc3d_bwd_f32(const float* x, const float* kernel, const float* grad_out, float* grad_x,
                                float* grad_kernel, int B, const int32_t* in_shape, int Cin, int Cout,
                                const int32_t* ksize, const int32_t* strides, int feature_order, int64_t p0,
                                int64_t p_count, void* stream) {
  NRT_REQUIRE(x && kernel && grad_out && in_shape && ksize && strides && (grad_x || grad_kernel), NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 0 && Cin >= 1 && Cout >= 1, NRT_E_ARG, "bad B/Cin/Cout");
  NRT_REQUIRE(feature_order == 0 || feature_order == 1, NRT_E_ARG, "feature_order must be 0 or 1");
  LcGeo g;
  g.B = B; g.Cin = Cin; g.Cout = Cout; g.feature_order = feature_order; g.activation = 0;
  g.P = 1; g.x_batch = Cin;
  int64_t F = Cin;
  for (int d = 0; d < 3; ++d) {
    g.I[d] = in_shape[d]; g.K[d] = ksize[d]; g.St[d] = strides[d];
    NRT_REQUIRE(g.I[d] >= 1 && g.K[d] >= 1 && g.St[d] >= 1 && g.K[d] <= g.I[d], NRT_E_ARG, "bad geometry at axis %d", d);
    g.O[d] = (g.I[d] - g.K[d]) / g.St[d] + 1;
    g.P *= g.O[d]; g.x_batch *= g.I[d]; F *= g.K[d];
  }
  NRT_REQUIRE(F <= 8192 && g.x_batch <= 0x7fffffffLL, NRT_E_SIZE, "patch or input too large");
  g.F = (int)F;
  NRT_REQUIRE(p0 >= 0 && p_count >= 0 && p0 + p_count <= g.P, NRT_E_ARG, "positions out of range");
  g.p0 = p0; g.pn = p_count;
  const int cq = Cout / 4;
  NRT_REQUIRE(Cout % 4 == 0 && cq <= 32 && (cq & (cq - 1)) == 0 && aligned16(kernel) && aligned16(grad_out) &&
              (!grad_kernel || aligned16(grad_kernel)), NRT_E_ARG,
              "lc3d backward is built for Cout in {4,8,16,32,64,128} and 16-byte aligned buffers");
  if (B == 0 || p_count == 0) return NRT_OK;
  int cq_log2 = 0;
  while ((1 << cq_log2) < cq) ++cq_log2;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = (int)imin64((p_count + 7) / 8, (int64_t)sm_count() * 8);
  const size_t smem = (size_t)g.F * sizeof(int);
  int b = 0;
  while (b < B) {
    const int left = B - b;
    const int acc = b > 0;
    if (left >= 4) { lc3d_bwd_kernel<4><<<grid, 256, smem, st>>>(x, kernel, grad_out, grad_x, grad_kernel, g, b, cq_log2, acc); b += 4; }
    else if (left >= 2) { lc3d_bwd_kernel<2><<<grid, 256, smem, st>>>(x, kernel, grad_out, grad_x, grad_kernel, g, b, cq_log2, acc); b += 2; }
    else { lc3d_bwd_kernel<1><<<grid, 256, smem, st>>>(x, kernel, grad_out, grad_x, grad_kernel, g, b, cq_log2, acc); b += 1; }
    int rc = check_launch("lc3d_bwd_kernel");
    if (rc != NRT_OK) return rc;
  }
  return NRT_OK;
}
