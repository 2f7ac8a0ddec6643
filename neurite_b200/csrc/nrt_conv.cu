// nrt_conv.cu -- separable 1-D convolution passes (GaussianBlur) and nearest re-indexing along an
// axis (Subsample): the stages either side of the warp in the synthesis pipeline (SURVEY.md 8f-4).
//
// Reference: neurite/tf/utils/utils.py:665-751 separable_conv (tf.nn.convolution = cross-
// correlation of every feature map with a 1-D kernel along one spatial axis, zero 'SAME' padding
// or 'VALID'), utils.py:581-662 gaussian_kernel, layers.py:251-364 GaussianBlur,
// utils.py:754-826 subsample_axis.
//
// A tensor [B, *space, C] seen from axis a is [outer, L, inner] with inner = prod(space[a+1:]) * C
// contiguous.  One pass reads and writes every element once (8 B per element is the roofline
// of a pass); the taps come out of a shared-memory tile:
//   * inner >= 32 ("column" pass): 128 (float4) or 32 inner elements x 64 outputs per CTA, every
//     thread slides a register window of outputs down the tile (8 shared loads per 32-64 FMAs);
//   * inner <  32 ("row" pass, e.g. the last axis of a single-channel volume): a flat 2048-output
//     segment + halo per CTA, row ends handled per tap;
//   * strides / dilations / huge kernels: one thread per output, taps from global memory.
// Accumulation is tap-ascending fp32 FMA; TF's order is unspecified (1e-5 tolerance).
#include "nrt_common.cuh"

namespace nrt {
namespace {

struct ConvArgs {
  const float* x;
  float* out;
  const float* k;      // device [K]
  int64_t outer, L, inner, L_out;
  int K, stride, dil, pad_before;
};

constexpr int kColTL = 64;     // outputs along L per CTA
constexpr int kColRL = 8;      // outputs per thread

// grid.x = outer * l_tiles * i_tiles (i fastest), block (32, 8), smem (kColTL + Kp - 1) * 32 + Kp floats
__global__ void __launch_bounds__(256) sepconv_col_kernel(const ConvArgs a, int Kp, int i_tiles, int l_tiles) {
  extern __shared__ float smem[];
  const int rows = kColTL + Kp - 1;
  float* sm = smem;                 // [rows][32]
  float* ks = smem + rows * 32;     // [Kp], zero padded
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;

  int64_t blk = blockIdx.x;
  const int it = (int)(blk % i_tiles);
  blk /= i_tiles;
  const int lt = (int)(blk % l_tiles);
  const int64_t o = blk / l_tiles;
  const int64_t i = (int64_t)it * 32 + tx;
  const int64_t l0 = (int64_t)lt * kColTL;
  const bool iok = i < a.inner;

  for (int j = tid; j < Kp; j += 256) ks[j] = j < a.K ? a.k[j] : 0.f;
  const float* xo = a.x + o * a.L * a.inner + i;
  for (int r = ty; r < rows; r += 8) {
    const int64_t lg = l0 - a.pad_before + r;
    sm[r * 32 + tx] = (iok && lg >= 0 && lg < a.L) ? ld_stream_f(xo + lg * a.inner) : 0.f;
  }
  __syncthreads();

  float acc[kColRL];
#pragma unroll
  for (int r = 0; r < kColRL; ++r) acc[r] = 0.f;
  const float* col = sm + (ty * kColRL) * 32 + tx;
  float v[kColRL + 7];
#pragma unroll
  for (int u = 0; u < 7; ++u) v[u] = col[u * 32];
  for (int c = 0; c < Kp; c += 8) {
#pragma unroll
    for (int u = 7; u < kColRL + 7; ++u) v[u] = col[(c + u) * 32];
    const float4 k0 = *reinterpret_cast<const float4*>(ks + c);
    const float4 k1 = *reinterpret_cast<const float4*>(ks + c + 4);
    const float kk[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int r = 0; r < kColRL; ++r) acc[r] = fmaf(kk[jj], v[r + jj], acc[r]);
#pragma unroll
    for (int u = 0; u < 7; ++u) v[u] = v[u + 8];
  }
  if (!iok) return;
  float* oo = a.out + o * a.L_out * a.inner + i;
#pragma unroll
  for (int r = 0; r < kColRL; ++r) {
    const int64_t l = l0 + ty * kColRL + r;
    if (l < a.L_out) st_stream_f(oo + l * a.inner, acc[r]);
  }
}


// float4 variant of the column pass: 128 inner elements x kColTL outputs per CTA, so every row of the
// tile is one 512-byte burst (the 32-wide tile reads 128-byte pieces 170 KB apart).  Needs
// inner % 4 == 0 and 16-byte aligned tensors.  block (32, 8); thread = 4 inner x kColRL outputs.
__global__ void __launch_bounds__(256) sepconv_col4_kernel(const ConvArgs a, int Kp, int i_tiles, int l_tiles) {
  extern __shared__ __align__(16) float smem[];
  const int rows = kColTL + Kp - 1;
  float4* sm = reinterpret_cast<float4*>(smem);        // [rows][32] float4
  float* ks = smem + rows * 128;                       // [Kp], zero padded
  const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;

  int64_t blk = blockIdx.x;
  const int it = (int)(blk % i_tiles);
  blk /= i_tiles;
  const int lt = (int)(blk % l_tiles);
  const int64_t o = blk / l_tiles;
  const int64_t i = (int64_t)it * 128 + tx * 4;
  const int64_t l0 = (int64_t)lt * kColTL;
  const bool iok = i < a.inner;                        // inner % 4 == 0: a float4 is all in or all out

  for (int j = tid; j < Kp; j += 256) ks[j] = j < a.K ? a.k[j] : 0.f;
  const float* xo = a.x + o * a.L * a.inner + i;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r = ty; r < rows; r += 8) {
    const int64_t lg = l0 - a.pad_before + r;
    sm[r * 32 + tx] = (iok && lg >= 0 && lg < a.L) ? ld_stream_f4(reinterpret_cast<const float4*>(xo + lg * a.inner)) : zero4;
  }
  __syncthreads();

  float4 acc[kColRL];
#pragma unroll
  for (int r = 0; r < kColRL; ++r) acc[r] = zero4;
  const float4* col = sm + (ty * kColRL) * 32 + tx;
  float4 v[kColRL + 7];
#pragma unroll
  for (int u = 0; u < 7; ++u) v[u] = col[u * 32];
  for (int c = 0; c < Kp; c += 8) {
#pragma unroll
    for (int u = 7; u < kColRL + 7; ++u) v[u] = col[(c + u) * 32];
    const float4 k0 = *reinterpret_cast<const float4*>(ks + c);
    const float4 k1 = *reinterpret_cast<const float4*>(ks + c + 4);
    const float kk[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
      for (int r = 0; r < kColRL; ++r) {
        acc[r].x = fmaf(kk[jj], v[r + jj].x, acc[r].x);
        acc[r].y = fmaf(kk[jj], v[r + jj].y, acc[r].y);
        acc[r].z = fmaf(kk[jj], v[r + jj].z, acc[r].z);
        acc[r].w = fmaf(kk[jj], v[r + jj].w, acc[r].w);
      }
#pragma unroll
    for (int u = 0; u < 7; ++u) v[u] = v[u + 8];
  }
  if (!iok) return;
  float* oo = a.out + o * a.L_out * a.inner + i;
#pragma unroll
  for (int r = 0; r < kColRL; ++r) {
    const int64_t l = l0 + ty * kColRL + r;
    if (l < a.L_out) st_stream_f4(reinterpret_cast<float4*>(oo + l * a.inner), acc[r]);
  }
}

constexpr int kRowTP = 2048;   // output positions per CTA
// The tensor is treated as one flat array of rows of rowlen = L * inner elements; a CTA takes kRowTP
// consecutive output positions (any number of rows, rows may straddle CTAs) plus the halo before
// and after, and each tap checks that it stays inside the output's own row (zero padding).
// Outputs far enough from both row ends skip the checks.  stride 1, L_out == L ('SAME') only.
// grid.x = ceil(outer * rowlen / kRowTP); smem kRowTP + (K-1)*dil*inner + K floats
__global__ void __launch_bounds__(256) sepconv_row_kernel(const ConvArgs a) {
  extern __shared__ float smem[];
  const int sp = (int)a.inner * a.dil;                 // tap spacing in elements
  const int halo = (a.K - 1) * sp;
  const int before = a.pad_before * (int)a.inner;      // elements of halo in front of an output
  float* sm = smem;                                    // [kRowTP + halo]
  float* ks = smem + kRowTP + halo;
  const int64_t rowlen = a.L * a.inner, total = a.outer * rowlen;
  const int64_t p0 = (int64_t)blockIdx.x * kRowTP;
  for (int j = threadIdx.x; j < a.K; j += 256) ks[j] = a.k[j];
  // stage [p0 - before, p0 + kRowTP + halo - before): 32-bit indices relative to one 64-bit base
  const float* src = a.x + (p0 - before);
  const int e_lo = p0 >= before ? 0 : (int)(before - p0);                                   // first staged element inside the tensor
  const int64_t e_end = total - p0 + before;
  const int e_hi = e_end < (int64_t)(kRowTP + halo) ? (int)e_end : kRowTP + halo;           // one past the last
  for (int e = threadIdx.x; e < kRowTP + halo; e += 256) sm[e] = (e >= e_lo && e < e_hi) ? ld_stream_f(src + e) : 0.f;
  __syncthreads();
  // warp w owns local positions [256 w, 256 w + 256): lane + 32 u, u < 8 (conflict-free shared loads, one
  // tap weight per 8 FMAs).  The main loop ignores row ends; the few outputs within a kernel radius of a
  // row end (6 of 224 for a 7-tap blur) are recomputed with per-tap checks afterwards.
  const int lane = threadIdx.x & 31, wbase = (threadIdx.x >> 5) * 256;
  const int rl = (int)rowlen;
  int orow = (int)((p0 + wbase + lane) % rowlen);       // position of output u = 0 inside its row
  const float* base = sm + wbase + lane;
  float acc[8];
#pragma unroll
  for (int u = 0; u < 8; ++u) acc[u] = 0.f;
#pragma unroll 2
  for (int j = 0; j < a.K; ++j) {
    const float kj = ks[j];
#pragma unroll
    for (int u = 0; u < 8; ++u) acc[u] = fmaf(kj, base[u * 32 + j * sp], acc[u]);
  }
  const int64_t left = total - p0 - wbase - lane;       // outputs from this lane's first one to the end of the tensor
  const int nleft = left > 256 ? 256 : (int)left;       // (may be <= 0)
  float* op = a.out + p0 + wbase + lane;
  const int step = 32 % rl;                             // orow advances by 32 (mod rowlen) per u
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const bool interior = (orow >= before) && (orow - before + halo < rl);
    float r = acc[u];
    if (!interior) {
      r = 0.f;
#pragma unroll 1
      for (int j = 0; j < a.K; ++j) {
        const int t = orow - before + j * sp;                          // tap position inside the row
        if ((unsigned)t < (unsigned)rl) r = fmaf(ks[j], base[u * 32 + j * sp], r);
      }
    }
    if (u * 32 < nleft) st_stream_f(op + u * 32, r);
    orow += step;
    if (orow >= rl) orow -= rl;
  }
}

__global__ void sepconv_generic_kernel(const ConvArgs a) {
  const int64_t total = a.outer * a.L_out * a.inner;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e % a.inner;
    const int64_t t = e / a.inner;
    const int64_t l = t % a.L_out, o = t / a.L_out;
    const float* xo = a.x + o * a.L * a.inner + i;
    float acc = 0.f;
    for (int j = 0; j < a.K; ++j) {
      const int64_t lg = l * a.stride - a.pad_before + (int64_t)j * a.dil;
      if (lg >= 0 && lg < a.L) acc = fmaf(__ldg(a.k + j), __ldg(xo + lg * a.inner), acc);
    }
    a.out[e] = acc;
  }
}


// out[o, l, i] = x[o, idx[l], i]   (tf.gather along an axis, utils.py:818-823)
__global__ void gather_axis_kernel(const float* x, const int32_t* idx, float* out, int64_t outer, int64_t L,
                                   int64_t inner, int64_t L_out) {
  const int64_t total = outer * L_out * inner;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e % inner;
    const int64_t t = e / inner;
    const int64_t l = t % L_out, o = t / L_out;
    const int64_t src = min(max((int64_t)idx[l], (int64_t)0), L - 1);
    out[e] = __ldg(x + (o * L + src) * inner + i);
  }
}

}  // namespace
}  // namespace nrt

using namespace nrt;

extern "C" {

int nrt_sepconv_axis_f32(const float* x, float* out, int64_t outer, int64_t L, int64_t inner, const float* kernel,
                         int K, int stride, int dilation, int pad_before, int64_t L_out, void* stream) {
  NRT_REQUIRE(x && out && kernel, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(x != out, NRT_E_ARG, "in-place convolution is not supported");
  NRT_REQUIRE(outer >= 0 && L >= 1 && inner >= 1 && L_out >= 0, NRT_E_ARG, "bad outer/L/inner/L_out");
  NRT_REQUIRE(K >= 1 && stride >= 1 && dilation >= 1 && pad_before >= 0, NRT_E_ARG, "bad K/stride/dilation/pad");
  const int64_t total = outer * L_out * inner;
  if (total == 0) return NRT_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ConvArgs a{x, out, kernel, outer, L, inner, L_out, K, stride, dilation, pad_before};
  const bool force_generic = env_int("NRT_CONV_GENERIC", 0) != 0;
  const int Kp = (K + 7) & ~7;
  const size_t col_smem = ((size_t)(kColTL + Kp - 1) * 32 + Kp) * sizeof(float);
  const int64_t halo = (int64_t)(K - 1) * dilation * inner;
  const size_t row_smem = (size_t)(kRowTP + halo + K) * sizeof(float);
  if (!force_generic && stride == 1 && dilation == 1 && inner >= 32) {
    const bool vec_ok = (inner % 4 == 0) && aligned16(x) && aligned16(out);
    const size_t col4_smem = ((size_t)(kColTL + Kp - 1) * 128 + Kp) * sizeof(float);
    if (vec_ok && col4_smem <= 48 * 1024) {
      const int64_t i_tiles = (inner + 127) / 128, l_tiles = (L_out + kColTL - 1) / kColTL;
      const int64_t nblk = outer * i_tiles * l_tiles;
      NRT_REQUIRE(nblk <= 2147483647LL, NRT_E_SIZE, "tensor too large for one launch");
      sepconv_col4_kernel<<<(unsigned)nblk, dim3(32, 8), col4_smem, st>>>(a, Kp, (int)i_tiles, (int)l_tiles);
      return check_launch("sepconv_col4_kernel");
    }
    if (col_smem <= 48 * 1024) {
      const int64_t i_tiles = (inner + 31) / 32, l_tiles = (L_out + kColTL - 1) / kColTL;
      const int64_t nblk = outer * i_tiles * l_tiles;
      NRT_REQUIRE(nblk <= 2147483647LL, NRT_E_SIZE, "tensor too large for one launch");
      sepconv_col_kernel<<<(unsigned)nblk, dim3(32, 8), col_smem, st>>>(a, Kp, (int)i_tiles, (int)l_tiles);
      return check_launch("sepconv_col_kernel");
    }
  }
  if (!force_generic && stride == 1 && inner < 32 && L_out == L && row_smem <= 48 * 1024 && L * inner < (1LL << 30)) {
    const int64_t nblk = (outer * L * inner + kRowTP - 1) / kRowTP;
    NRT_REQUIRE(nblk <= 2147483647LL, NRT_E_SIZE, "tensor too large for one launch");
    sepconv_row_kernel<<<(unsigned)nblk, 256, row_smem, st>>>(a);
    return check_launch("sepconv_row_kernel");
  }
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 32);
  sepconv_generic_kernel<<<grid, 256, 0, st>>>(a);
  return check_launch("sepconv_generic_kernel");
}

int nrt_gather_axis_f32(const float* x, const int32_t* index, float* out, int64_t outer, int64_t L, int64_t inner,
                        int64_t L_out, void* stream) {
  NRT_REQUIRE(x && index && out, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(outer >= 0 && L >= 1 && inner >= 1 && L_out >= 0, NRT_E_ARG, "bad outer/L/inner/L_out");
  const int64_t total = outer * L_out * inner;
  if (total == 0) return NRT_OK;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 32);
  gather_axis_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, index, out, outer, L, inner, L_out);
  return check_launch("gather_axis_kernel");
}

}  // extern "C"
