// nrt_interp.cu -- N-D gridded interpolation for sm_90a:
//   nrt_interpn_f32  (explicit loc tensor)      reference utils.py:73-220
//   nrt_warp_f32     (identity grid + flow)     voxelmorph SpatialTransformer contract
//   nrt_resize_f32   (in-kernel linspace grid)  reference utils.py:223-265, layers.py:154-181
//
// Two kernel families:
//   * generic gather kernels (any D in 1..3, any C, linear/nearest): one thread per
//     (output point, 4-channel chunk); corners read through L1/L2 with __ldg.
//   * warp3d_tile_kernel (D=3, C=1): the hot kernel of BASELINE.json.  One CTA per
//     TZxTYx32 output tile; the flow tile and the bounding source box (tile + halo) are
//     staged into shared memory by two TMA tensor loads completing on one mbarrier; the
//     8-corner gather runs from shared memory (bank-conflict bound instead of L1-sector
//     bound for incoherent flows).  Any corner outside the staged box falls back, per
//     voxel, to the global gather, so results never depend on the halo.
//
// Arithmetic is bit-faithful to the reference's unfused TF ops: every multiply and add is
// a separate fp32 rounding (__fmul_rn/__fadd_rn), corner order is itertools.product order.
#include <string.h>

#include "nrt_interp.cuh"

namespace nrt {


// ---------------------------------------------------------------------------------------
// generic kernels
// ---------------------------------------------------------------------------------------
template <int D, int VEC, int METHOD>
__global__ void __launch_bounds__(256)
interpn_kernel(const float* __restrict__ vol, Geo g, const float* __restrict__ loc_t,
               int64_t n_out, float* __restrict__ out) {
  const int cv_n = VEC == 4 ? g.C / 4 : 1;
  const int64_t total = n_out * cv_n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pt = t / cv_n;
    const int c0 = (int)(t - pt * cv_n) * VEC;
    float loc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) loc[d] = __ldg(loc_t + pt * D + d);
    sample_store<D, VEC, METHOD>(vol, g, loc, c0, out + pt * g.C);
  }
}

struct WarpGeo {
  Geo g;
  int out_z0, out_n0;   // produced planes of axis 0
  int64_t src_batch_stride, out_vox;   // elements per batch item of vol; voxels per batch item of out
  int64_t flow_bstride, out_bstride;   // elements between batch items of flow / out (dense: out_vox*D, out_vox*C)
  int B;
};

template <int D, int VEC, int METHOD>
__global__ void __launch_bounds__(256)
warp_generic_kernel(const float* __restrict__ vol, const float* __restrict__ flow,
                    float* __restrict__ out, WarpGeo w) {
  const Geo& g = w.g;
  const int cv_n = VEC == 4 ? g.C / 4 : 1;
  const int64_t total = (int64_t)w.B * w.out_vox * cv_n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pv = t / cv_n;                       // (b, voxel)
    const int c0 = (int)(t - pv * cv_n) * VEC;
    const int b = (int)(pv / w.out_vox);
    int rem = (int)(pv - (int64_t)b * w.out_vox);
    int coord[D];
#pragma unroll
    for (int d = D - 1; d >= 1; --d) { coord[d] = rem % g.S[d]; rem /= g.S[d]; }
    coord[0] = rem + w.out_z0;
    float loc[D];
    const int64_t vox = pv - (int64_t)b * w.out_vox;
    const float* fl = flow + (size_t)b * w.flow_bstride + vox * D;
#pragma unroll
    for (int d = 0; d < D; ++d) loc[d] = __fadd_rn((float)coord[d], __ldg(fl + d));
    sample_store<D, VEC, METHOD>(vol + (size_t)b * w.src_batch_stride, g, loc, c0,
                                 out + (size_t)b * w.out_bstride + vox * g.C);
  }
}

struct ResizeGeo {
  Geo g;
  int M[3];          // full output extent
  float delta[3];    // fp32 (S-1)/(M-1)
  int out_z0, out_n0;
  int64_t src_batch_stride, out_vox;
  int B;
};

template <int D, int VEC, int METHOD>
__global__ void __launch_bounds__(256)
resize_kernel(const float* __restrict__ vol, float* __restrict__ out, ResizeGeo w) {
  const Geo& g = w.g;
  const int cv_n = VEC == 4 ? g.C / 4 : 1;
  const int64_t total = (int64_t)w.B * w.out_vox * cv_n;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t pv = t / cv_n;
    const int c0 = (int)(t - pv * cv_n) * VEC;
    const int b = (int)(pv / w.out_vox);
    int rem = (int)(pv - (int64_t)b * w.out_vox);
    int coord[D];
#pragma unroll
    for (int d = D - 1; d >= 1; --d) { coord[d] = rem % w.M[d]; rem /= w.M[d]; }
    coord[0] = rem + w.out_z0;
    float loc[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      // tf.linspace(0, S-1, M): endpoints exact, interior 0 + delta*i  (utils.py:259)
      const int i = coord[d];
      loc[d] = (i == w.M[d] - 1 && w.M[d] > 1) ? (float)(g.S[d] - 1) : __fmul_rn(w.delta[d], (float)i);
    }
    sample_store<D, VEC, METHOD>(vol + (size_t)b * w.src_batch_stride, g, loc, c0, out + pv * g.C);
  }
}

// ---------------------------------------------------------------------------------------
// resize3d_kernel: D=3 zoom.  Sample coordinates are separable (one linspace per axis), so a
// CTA first builds per-axis tables {offset(i0), offset(i1), wlo, whi} for its output tile in
// shared memory (axis_linear on the linspace value: identical arithmetic to the generic
// path), then every thread combines three table entries per voxel: no per-voxel floor/clip,
// no div/mod, corner setup shared by all channels.
// ---------------------------------------------------------------------------------------
struct AxisEntry { int o0, o1; float wlo, whi; };

// CT = compile-time channel count (1..4: unrolled, immediate load offsets) or 0 = run-time C
// TZ = output planes marched by one CTA (8, 16 or 32: fewer table builds and source-plane reloads per voxel)
template <int METHOD, int CT, int TZ = 8>
__global__ void __launch_bounds__(256)
resize3d_kernel(const float* __restrict__ vol, float* __restrict__ out, ResizeGeo w, int ntz, int nty, int ntx) {
  constexpr int TY = 8, TX = 32;
  __shared__ AxisEntry s_ax[TZ + TY + TX];
  const Geo& g = w.g;
  const int C = CT > 0 ? CT : g.C;
  int tile = blockIdx.x;
  const int tx = tile % ntx; tile /= ntx;
  const int ty = tile % nty; tile /= nty;
  const int tz = tile % ntz;
  const int b = tile / ntz;
  const int x0 = tx * TX, y0 = ty * TY, z0 = tz * TZ;            // z0 relative to the produced slab
  if (threadIdx.x < TZ + TY + TX) {
    const int t = threadIdx.x;
    const int d = t < TZ ? 0 : (t < TZ + TY ? 1 : 2);
    const int i = d == 0 ? w.out_z0 + z0 + t : (d == 1 ? y0 + (t - TZ) : x0 + (t - TZ - TY));
    const int stride = d == 0 ? g.S[1] * g.S[2] * C : (d == 1 ? g.S[2] * C : C);
    AxisEntry e;
    if (i < w.M[d]) {
      // tf.linspace(0, S-1, M): endpoints exact, interior 0 + delta*i  (utils.py:259)
      const float loc = (i == w.M[d] - 1 && w.M[d] > 1) ? (float)(g.S[d] - 1) : __fmul_rn(w.delta[d], (float)i);
      if (METHOD == NRT_LINEAR) {
        const Axis a = axis_linear(loc, (float)(g.S[d] - 1), g.S[d] - 1);
        e.o0 = a.i0 * stride; e.o1 = a.i1 * stride; e.wlo = a.wlo; e.whi = a.whi;
      } else {
        e.o0 = e.o1 = axis_nearest(loc, g.S[d] - 1) * stride; e.wlo = 1.f; e.whi = 0.f;
      }
    } else {
      e.o0 = e.o1 = 0; e.wlo = e.whi = 0.f;
    }
    s_ax[t] = e;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int ox = x0 + lane, oy = y0 + wid;
  // (C = 3 rows exchanged through shared memory for coalesced 128-byte stores were tried: the warp syncs cost more
  // than the write sectors they saved)
  if (oy >= w.M[1] || ox >= w.M[2]) return;
  const AxisEntry ey = s_ax[TZ + wid], ex = s_ax[TZ + TY + lane];
  const float* volb = vol + (size_t)b * w.src_batch_stride;
  float* outb = out + ((size_t)b * w.out_vox + ((size_t)z0 * w.M[1] + oy) * w.M[2] + ox) * C;
  const size_t plane = (size_t)w.M[1] * w.M[2] * C;
  if (METHOD == NRT_LINEAR && CT > 0) {
    // March along z keeping the 2 x 4 corner values of the two source planes in registers.  The
    // z entry is the same for the whole warp, so "same plane as before" / "old upper plane is the
    // new lower plane" are uniform branches: an upsampling zoom re-reads a source plane only when
    // the output plane crosses into the next source cell (zoom 2: 12 loads per 2 outputs at C = 3
    // instead of 48).
    const float* q00 = volb + ey.o0 + ex.o0; const float* q01 = volb + ey.o0 + ex.o1;
    const float* q10 = volb + ey.o1 + ex.o0; const float* q11 = volb + ey.o1 + ex.o1;
    constexpr int CN = CT > 0 ? CT : 1;
    float lo[4][CN], hi[4][CN];
    int cur0 = -1, cur1 = -1;
#pragma unroll 1
    for (int z = 0; z < TZ; ++z, outb += plane) {
      if (z0 + z >= w.out_n0) break;
      const AxisEntry ez = s_ax[z];
      if (ez.o0 != cur0) {
        if (ez.o0 == cur1) {
#pragma unroll
          for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int c = 0; c < CT; ++c) lo[q][c] = hi[q][c];
        } else {
#pragma unroll
          for (int c = 0; c < CT; ++c) {
            lo[0][c] = __ldg(q00 + ez.o0 + c); lo[1][c] = __ldg(q01 + ez.o0 + c);
            lo[2][c] = __ldg(q10 + ez.o0 + c); lo[3][c] = __ldg(q11 + ez.o0 + c);
          }
        }
        cur0 = ez.o0;
      }
      if (ez.o1 != cur1) {
        if (ez.o1 == cur0) {
#pragma unroll
          for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int c = 0; c < CT; ++c) hi[q][c] = lo[q][c];
        } else {
#pragma unroll
          for (int c = 0; c < CT; ++c) {
            hi[0][c] = __ldg(q00 + ez.o1 + c); hi[1][c] = __ldg(q01 + ez.o1 + c);
            hi[2][c] = __ldg(q10 + ez.o1 + c); hi[3][c] = __ldg(q11 + ez.o1 + c);
          }
        }
        cur1 = ez.o1;
      }
      const float w00 = __fmul_rn(ez.wlo, ey.wlo), w01 = __fmul_rn(ez.wlo, ey.whi);
      const float w10 = __fmul_rn(ez.whi, ey.wlo), w11 = __fmul_rn(ez.whi, ey.whi);
      const float k0 = __fmul_rn(w00, ex.wlo), k1 = __fmul_rn(w00, ex.whi), k2 = __fmul_rn(w01, ex.wlo), k3 = __fmul_rn(w01, ex.whi);
      const float k4 = __fmul_rn(w10, ex.wlo), k5 = __fmul_rn(w10, ex.whi), k6 = __fmul_rn(w11, ex.wlo), k7 = __fmul_rn(w11, ex.whi);
      float res[CN];
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        float r = __fadd_rn(0.f, __fmul_rn(k0, lo[0][c]));
        r = __fadd_rn(r, __fmul_rn(k1, lo[1][c]));
        r = __fadd_rn(r, __fmul_rn(k2, lo[2][c]));
        r = __fadd_rn(r, __fmul_rn(k3, lo[3][c]));
        r = __fadd_rn(r, __fmul_rn(k4, hi[0][c]));
        r = __fadd_rn(r, __fmul_rn(k5, hi[1][c]));
        r = __fadd_rn(r, __fmul_rn(k6, hi[2][c]));
        r = __fadd_rn(r, __fmul_rn(k7, hi[3][c]));
        res[c] = r;
      }
      if (CT == 4) {
        *reinterpret_cast<float4*>(outb) = make_float4(res[0], res[1], res[2], res[3]);     // 16-byte aligned: 4 floats per voxel
      } else if (CT == 2) {
        *reinterpret_cast<float2*>(outb) = make_float2(res[0], res[1]);
      } else {
#pragma unroll
        for (int c = 0; c < CT; ++c) outb[c] = res[c];
      }
    }
    return;
  }
  if (METHOD == NRT_LINEAR && CT > 0) return;      // (handled above)
#pragma unroll 2
  for (int z = 0; z < TZ; ++z, outb += plane) {
    if (z0 + z >= w.out_n0) break;
    const AxisEntry ez = s_ax[z];
    if (METHOD == NRT_LINEAR) {
      const int b00 = ez.o0 + ey.o0, b01 = ez.o0 + ey.o1, b10 = ez.o1 + ey.o0, b11 = ez.o1 + ey.o1;
      const float w00 = __fmul_rn(ez.wlo, ey.wlo), w01 = __fmul_rn(ez.wlo, ey.whi);
      const float w10 = __fmul_rn(ez.whi, ey.wlo), w11 = __fmul_rn(ez.whi, ey.whi);
      const float k0 = __fmul_rn(w00, ex.wlo), k1 = __fmul_rn(w00, ex.whi), k2 = __fmul_rn(w01, ex.wlo), k3 = __fmul_rn(w01, ex.whi);
      const float k4 = __fmul_rn(w10, ex.wlo), k5 = __fmul_rn(w10, ex.whi), k6 = __fmul_rn(w11, ex.wlo), k7 = __fmul_rn(w11, ex.whi);
      const float* p0 = volb + b00 + ex.o0; const float* p1 = volb + b00 + ex.o1;
      const float* p2 = volb + b01 + ex.o0; const float* p3 = volb + b01 + ex.o1;
      const float* p4 = volb + b10 + ex.o0; const float* p5 = volb + b10 + ex.o1;
      const float* p6 = volb + b11 + ex.o0; const float* p7 = volb + b11 + ex.o1;
#pragma unroll
      for (int c = 0; c < C; ++c) {
        float r = __fadd_rn(0.f, __fmul_rn(k0, __ldg(p0 + c)));
        r = __fadd_rn(r, __fmul_rn(k1, __ldg(p1 + c)));
        r = __fadd_rn(r, __fmul_rn(k2, __ldg(p2 + c)));
        r = __fadd_rn(r, __fmul_rn(k3, __ldg(p3 + c)));
        r = __fadd_rn(r, __fmul_rn(k4, __ldg(p4 + c)));
        r = __fadd_rn(r, __fmul_rn(k5, __ldg(p5 + c)));
        r = __fadd_rn(r, __fmul_rn(k6, __ldg(p6 + c)));
        r = __fadd_rn(r, __fmul_rn(k7, __ldg(p7 + c)));
        outb[c] = r;
      }
    } else {
      const float* p0 = volb + ez.o0 + ey.o0 + ex.o0;
#pragma unroll
      for (int c = 0; c < C; ++c) outb[c] = __ldg(p0 + c);
    }
  }
}

// ---------------------------------------------------------------------------------------
// resize3d_tile_kernel: the linear z-marching kernel with its SOURCE staged in shared memory.  resize3d_kernel issues
// its corner loads to L1/L2 when an output plane enters a new source cell and then waits ~600 cycles for them with
// 3 CTAs per SM: it is latency-bound.  An up-sampling zoom reads a SMALL source box per output tile -- 32 x 8 x 32
// outputs of a x2 zoom touch 18 x 6 x 18 source voxels -- so the CTA fetches that box with ONE TMA tensor load
// (coordinates from the tile's own table entries, extents = the largest box any tile needs, computed on the host
// with the same fp32 linspace arithmetic) and every corner read becomes a ~30-cycle LDS.
// A tile whose box would not fit the staged extents (cannot happen when host and device agree) or a zoom whose
// boxes are larger than the budget (down-sampling) takes resize3d_kernel.
// ---------------------------------------------------------------------------------------
// fp32 pair arithmetic (pack2 / fma2 in nrt_interp.cuh).  Bit-exactness: the reference's separately rounded ops are
// written as  a*b = fma(a, b, -0)  and  a+b = fma(a, 1, b)  with the identity operands (-0,-0) and (1,1) passed as
// kernel PARAMETERS (visible constants would be folded and the multiply and add re-fused into one rounding).
struct ResizeBox { int bz, by, bx; };            // staged source extents (bx already padded for the TMA alignment)

template <int CT, int TZ>
__global__ void __launch_bounds__(256)
resize3d_tile_kernel(const __grid_constant__ CUtensorMap tm_vol, const float* __restrict__ vol, float* __restrict__ out,
                     ResizeGeo w, ResizeBox bxs, int ntz, int nty, int ntx, int xalign) {
  constexpr int TY = 8, TX = 32;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_box = reinterpret_cast<float*>(smem_raw);                                     // [bz][by][bx][CT]
  const int box_elems = bxs.bz * bxs.by * bxs.bx * CT;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + (((size_t)box_elems * 4 + 15) & ~(size_t)15));
  int* s_lo = reinterpret_cast<int*>(bar + 1);                                           // box origin (source voxels)
  __shared__ AxisEntry s_ax[TZ + TY + TX];
  __shared__ int s_i[2][TZ + TY + TX];                                                   // i0 / i1 per table entry
  const Geo& g = w.g;
  int tile = blockIdx.x;
  const int tx = tile % ntx; tile /= ntx;
  const int ty = tile % nty; tile /= nty;
  const int tz = tile % ntz;
  const int b = tile / ntz;
  const int x0 = tx * TX, y0 = ty * TY, z0 = tz * TZ;            // z0 relative to the produced slab
  if (threadIdx.x == 0) { mbar_init(bar, 1); fence_mbar_init(); }
  if (threadIdx.x < TZ + TY + TX) {
    const int t = threadIdx.x;
    const int d = t < TZ ? 0 : (t < TZ + TY ? 1 : 2);
    const int i = d == 0 ? w.out_z0 + z0 + t : (d == 1 ? y0 + (t - TZ) : x0 + (t - TZ - TY));
    AxisEntry e;
    int i0 = -1, i1 = -1;
    if (i < w.M[d] && (d != 0 || z0 + t < w.out_n0)) {
      // tf.linspace(0, S-1, M): endpoints exact, interior 0 + delta*i  (utils.py:259)
      const float loc = (i == w.M[d] - 1 && w.M[d] > 1) ? (float)(g.S[d] - 1) : __fmul_rn(w.delta[d], (float)i);
      const Axis a = axis_linear(loc, (float)(g.S[d] - 1), g.S[d] - 1);
      i0 = a.i0; i1 = a.i1; e.wlo = a.wlo; e.whi = a.whi;
    } else {
      e.wlo = e.whi = 0.f;
    }
    e.o0 = e.o1 = 0;
    s_ax[t] = e; s_i[0][t] = i0; s_i[1][t] = i1;
  }
  __syncthreads();
  // box origin = first corner of the tile's first output per axis (linspace is monotonic); x aligned for the TMA
  if (threadIdx.x == 0) {
    int lo[3], ok = 1;
    const int first[3] = {0, TZ, TZ + TY}, count[3] = {TZ, TY, TX}, ext[3] = {bxs.bz, bxs.by, bxs.bx};
    for (int d = 0; d < 3; ++d) {
      lo[d] = s_i[0][first[d]];
      if (d == 2) lo[d] -= lo[d] % xalign;
      int hi = lo[d];
      for (int k = 0; k < count[d]; ++k) hi = max(hi, s_i[1][first[d] + k]);
      ok &= (hi - lo[d] + 1 <= ext[d]);
    }
    s_lo[0] = lo[0]; s_lo[1] = lo[1]; s_lo[2] = lo[2]; s_lo[3] = ok;
    if (ok) {
      mbar_expect_tx(bar, (uint32_t)(box_elems * sizeof(float)));
      tma_load_4d(s_box, &tm_vol, bar, lo[2] * CT, lo[1], lo[0], b);
    }
  }
  __syncthreads();
  const bool staged = s_lo[3] != 0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int ox = x0 + lane, oy = y0 + wid;
  // offsets of this thread's table entries: box-relative when staged, else into the global volume
  const int sz_ = staged ? bxs.by * bxs.bx * CT : g.S[1] * g.S[2] * CT;
  const int sy_ = staged ? bxs.bx * CT : g.S[2] * CT;
  const int lz = staged ? s_lo[0] : 0, ly = staged ? s_lo[1] : 0, lx = staged ? s_lo[2] : 0;
  if (staged) mbar_wait(bar, 0);
  if (oy >= w.M[1] || ox >= w.M[2]) return;
  const AxisEntry ey = s_ax[TZ + wid], ex = s_ax[TZ + TY + lane];
  const int y_o0 = (s_i[0][TZ + wid] - ly) * sy_, y_o1 = (s_i[1][TZ + wid] - ly) * sy_;
  const int x_o0 = (s_i[0][TZ + TY + lane] - lx) * CT, x_o1 = (s_i[1][TZ + TY + lane] - lx) * CT;
  const float* src = staged ? s_box : vol + (size_t)b * w.src_batch_stride;
  float* outb = out + ((size_t)b * w.out_vox + ((size_t)z0 * w.M[1] + oy) * w.M[2] + ox) * CT;
  const size_t plane = (size_t)w.M[1] * w.M[2] * CT;
  const float* q00 = src + y_o0 + x_o0; const float* q01 = src + y_o0 + x_o1;
  const float* q10 = src + y_o1 + x_o0; const float* q11 = src + y_o1 + x_o1;
  float lo[4][CT], hi[4][CT];
  int cur0 = -1, cur1 = -1;
#pragma unroll 1
  for (int z = 0; z < TZ; ++z, outb += plane) {
    if (z0 + z >= w.out_n0) break;
    const AxisEntry ez = s_ax[z];
    const int z_o0 = (s_i[0][z] - lz) * sz_, z_o1 = (s_i[1][z] - lz) * sz_;
    if (z_o0 != cur0) {
      if (z_o0 == cur1) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int c = 0; c < CT; ++c) lo[q][c] = hi[q][c];
      } else {
#pragma unroll
        for (int c = 0; c < CT; ++c) {
          lo[0][c] = q00[z_o0 + c]; lo[1][c] = q01[z_o0 + c];
          lo[2][c] = q10[z_o0 + c]; lo[3][c] = q11[z_o0 + c];
        }
      }
      cur0 = z_o0;
    }
    if (z_o1 != cur1) {
      if (z_o1 == cur0) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int c = 0; c < CT; ++c) hi[q][c] = lo[q][c];
      } else {
#pragma unroll
        for (int c = 0; c < CT; ++c) {
          hi[0][c] = q00[z_o1 + c]; hi[1][c] = q01[z_o1 + c];
          hi[2][c] = q10[z_o1 + c]; hi[3][c] = q11[z_o1 + c];
        }
      }
      cur1 = z_o1;
    }
    const float w00 = __fmul_rn(ez.wlo, ey.wlo), w01 = __fmul_rn(ez.wlo, ey.whi);
    const float w10 = __fmul_rn(ez.whi, ey.wlo), w11 = __fmul_rn(ez.whi, ey.whi);
    const float k0 = __fmul_rn(w00, ex.wlo), k1 = __fmul_rn(w00, ex.whi), k2 = __fmul_rn(w01, ex.wlo), k3 = __fmul_rn(w01, ex.whi);
    const float k4 = __fmul_rn(w10, ex.wlo), k5 = __fmul_rn(w10, ex.whi), k6 = __fmul_rn(w11, ex.wlo), k7 = __fmul_rn(w11, ex.whi);
    float res[CT];
#pragma unroll
    for (int c = 0; c < CT; ++c) {
      float r = __fadd_rn(0.f, __fmul_rn(k0, lo[0][c]));
      r = __fadd_rn(r, __fmul_rn(k1, lo[1][c]));
      r = __fadd_rn(r, __fmul_rn(k2, lo[2][c]));
      r = __fadd_rn(r, __fmul_rn(k3, lo[3][c]));
      r = __fadd_rn(r, __fmul_rn(k4, hi[0][c]));
      r = __fadd_rn(r, __fmul_rn(k5, hi[1][c]));
      r = __fadd_rn(r, __fmul_rn(k6, hi[2][c]));
      r = __fadd_rn(r, __fmul_rn(k7, hi[3][c]));
      res[c] = r;
    }
    if (CT == 4) {
      *reinterpret_cast<float4*>(outb) = make_float4(res[0], res[1 % CT], res[2 % CT], res[3 % CT]);
    } else if (CT == 2) {
      *reinterpret_cast<float2*>(outb) = make_float2(res[0], res[1 % CT]);
    } else {
#pragma unroll
      for (int c = 0; c < CT; ++c) outb[c] = res[c];
    }
  }
}

// ---------------------------------------------------------------------------------------
// resize3d_pair_kernel: the voxel-pair kernel (two x positions per thread share the table reads and the z / y weights):
//   * corner reads are LDS with 32-bit offsets and immediate channel offsets, not generic loads through a pointer that
//     is shared OR global at run time (64-bit address arithmetic per load): the marching loop is a template on the
//     address space.
//   * the two source planes of a z cell live in two register sets tagged with the source plane they hold; entering
//     the next cell loads ONE plane into the set that is free and swaps the roles of the sets (two copies of the
//     arithmetic, selected by a CTA-uniform branch) instead of moving 24 registers from `hi` to `lo`.
//   * prologue: one thread derives the box origin from the tile's first / last output per axis (the linspace is
//     monotonic: no loop over the table, no second block barrier) and issues the TMA load while the other threads
//     build the tables; no dynamically indexed kernel parameters (they cost a 128-byte local-memory copy per thread).
// Same arithmetic and rounding order as resize3d_tile_kernel (bit-exact with the oracle); two x positions per thread
// are the halves of fp32 register pairs.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ Axis resize_axis(int S, int M, float delta, int i) {
  // tf.linspace(0, S-1, M): endpoints exact, interior 0 + delta*i  (utils.py:259)
  const float loc = (i == M - 1 && M > 1) ? (float)(S - 1) : __fmul_rn(delta, (float)i);
  return axis_linear(loc, (float)(S - 1), S - 1);
}

template <int CT>
__device__ __forceinline__ void resize_pair_emit(const f32x2 (&lo)[4][CT], const f32x2 (&hi)[4][CT], const f32x2 (&k)[8],
                                                 f32x2 negzero2, f32x2 one2, f32x2 zero2, float* __restrict__ outb,
                                                 bool has1) {
  float ra[CT], rb[CT];
#pragma unroll
  for (int c = 0; c < CT; ++c) {
    f32x2 r = fma2(fma2(k[0], lo[0][c], negzero2), one2, zero2);          // 0 + k0*v0
#pragma unroll
    for (int q = 1; q < 4; ++q) r = fma2(fma2(k[q], lo[q][c], negzero2), one2, r);
#pragma unroll
    for (int q = 0; q < 4; ++q) r = fma2(fma2(k[4 + q], hi[q][c], negzero2), one2, r);
    unpack2(r, ra[c], rb[c]);
  }
  if (!has1) {
#pragma unroll
    for (int c = 0; c < CT; ++c) outb[c] = ra[c];
  } else if (CT == 1) {
    *reinterpret_cast<float2*>(outb) = make_float2(ra[0], rb[0]);
  } else if (CT == 2) {
    *reinterpret_cast<float4*>(outb) = make_float4(ra[0], ra[1 % CT], rb[0], rb[1 % CT]);
  } else if (CT == 3) {
    *reinterpret_cast<float2*>(outb) = make_float2(ra[0], ra[1 % CT]);
    *reinterpret_cast<float2*>(outb + 2) = make_float2(ra[2 % CT], rb[0]);
    *reinterpret_cast<float2*>(outb + 4) = make_float2(rb[1 % CT], rb[2 % CT]);
  } else {
    *reinterpret_cast<float4*>(outb) = make_float4(ra[0], ra[1 % CT], ra[2 % CT], ra[3 % CT]);
    *reinterpret_cast<float4*>(outb + 4) = make_float4(rb[0], rb[1 % CT], rb[2 % CT], rb[3 % CT]);
  }
}

// One corner (CT channels) of both voxels of a pair -> packed registers.  SHARED: 32-bit shared-window byte addresses and
// ld.shared with the channel as an immediate offset (written as asm: left to itself the compiler keeps element indices
// and re-derives every address from the window base inside the loop); else global element pointers.
template <int OFF>
__device__ __forceinline__ float lds_imm(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(OFF));
  return v;
}
template <int CT, bool SHARED, typename AddrT>
__device__ __forceinline__ void resize_pair_corner(f32x2 (&dst)[CT], AddrT a, AddrT b) {
  if constexpr (SHARED) {
    dst[0] = pack2(lds_imm<0>(a), lds_imm<0>(b));
    if constexpr (CT > 1) dst[1] = pack2(lds_imm<4>(a), lds_imm<4>(b));
    if constexpr (CT > 2) dst[2] = pack2(lds_imm<8>(a), lds_imm<8>(b));
    if constexpr (CT > 3) dst[3] = pack2(lds_imm<12>(a), lds_imm<12>(b));
  } else {
#pragma unroll
    for (int c = 0; c < CT; ++c) dst[c] = pack2(a[c], b[c]);
  }
}

// SHARED: `sbox` = shared-window address of the staged box; else `src` = the batch item's volume in global memory.
// oa / ob = (y, x) corner offsets (elements) of the pair's two voxels at the first staged plane lz (0 for global),
// zs = z stride in elements.
template <int CT, int TZ, bool SHARED>
__device__ __forceinline__ void resize_pair_march(uint32_t sbox, const float* __restrict__ src, const int (&oa)[4],
                                                  const int (&ob)[4], int zs, int lz, const float2* __restrict__ s_w,
                                                  const int* __restrict__ s_i0, const int* __restrict__ s_i1, int nz,
                                                  float2 wy, f32x2 exlo, f32x2 exhi, float* __restrict__ outb,
                                                  size_t plane, bool has1, f32x2 negzero2, f32x2 one2) {
  using AddrT = typename std::conditional<SHARED, uint32_t, const float*>::type;
  const f32x2 zero2 = pack2(0.f, 0.f);
  AddrT pa[4], pb[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if constexpr (SHARED) { pa[q] = sbox + 4u * (uint32_t)oa[q]; pb[q] = sbox + 4u * (uint32_t)ob[q]; }
    else { pa[q] = src + oa[q]; pb[q] = src + ob[q]; }
  }
  const int zstep = SHARED ? zs * 4 : zs;                // bytes / elements per source plane
  f32x2 P[4][CT], Q[4][CT];
  int tagP = -1, tagQ = -1;                              // source plane held by either register set
#pragma unroll 1
  for (int z = 0; z < nz; ++z, outb += plane) {
    const float2 wz = s_w[z];
    const int i0 = s_i0[z], i1 = s_i1[z];
    // (lo, hi) = (P, Q) unless Q already holds the lower plane: then (Q, P).  CTA-uniform.
    const bool swapped = (tagQ == i0);
    const int needP = swapped ? i1 : i0, needQ = swapped ? i0 : i1;
    if (tagP != needP) {
      const int zo = (needP - lz) * zstep;
#pragma unroll
      for (int q = 0; q < 4; ++q) resize_pair_corner<CT, SHARED, AddrT>(P[q], pa[q] + zo, pb[q] + zo);
      tagP = needP;
    }
    if (tagQ != needQ) {
      const int zo = (needQ - lz) * zstep;
#pragma unroll
      for (int q = 0; q < 4; ++q) resize_pair_corner<CT, SHARED, AddrT>(Q[q], pa[q] + zo, pb[q] + zo);
      tagQ = needQ;
    }
    const float w00 = __fmul_rn(wz.x, wy.x), w01 = __fmul_rn(wz.x, wy.y);
    const float w10 = __fmul_rn(wz.y, wy.x), w11 = __fmul_rn(wz.y, wy.y);
    const f32x2 p00 = pack2(w00, w00), p01 = pack2(w01, w01), p10 = pack2(w10, w10), p11 = pack2(w11, w11);
    f32x2 k[8];
    k[0] = fma2(p00, exlo, negzero2); k[1] = fma2(p00, exhi, negzero2);
    k[2] = fma2(p01, exlo, negzero2); k[3] = fma2(p01, exhi, negzero2);
    k[4] = fma2(p10, exlo, negzero2); k[5] = fma2(p10, exhi, negzero2);
    k[6] = fma2(p11, exlo, negzero2); k[7] = fma2(p11, exhi, negzero2);
    if (swapped) resize_pair_emit<CT>(Q, P, k, negzero2, one2, zero2, outb, has1);
    else resize_pair_emit<CT>(P, Q, k, negzero2, one2, zero2, outb, has1);
  }
}

template <int CT, int TZ>
__global__ void __launch_bounds__(256)
resize3d_pair_kernel(const __grid_constant__ CUtensorMap tm_vol, const float* __restrict__ vol, float* __restrict__ out,
                     ResizeGeo w, ResizeBox bxs, int ntz, int nty, int ntx, int xalign, f32x2 negzero2, f32x2 one2,
                     int unstaged) {
  constexpr int TY = 16, TX = 32, NT = TZ + TY + TX;   // a warp = two rows of 16 x-pairs
  static_assert(NT < 255, "thread 255 issues the load, the threads below NT build the tables");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_box = reinterpret_cast<float*>(smem_raw);                                     // [bz][by][bx][CT]
  const int box_elems = bxs.bz * bxs.by * bxs.bx * CT;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + (((size_t)box_elems * 4 + 15) & ~(size_t)15));
  int* s_lo = reinterpret_cast<int*>(bar + 1);
  __shared__ float2 s_w[NT];                                                             // (wlo, whi) per table entry
  __shared__ int s_i[2][NT];                                                             // i0 / i1 per table entry
  const Geo& g = w.g;
  int tile = blockIdx.x;
  const int tx = tile % ntx; tile /= ntx;
  const int ty = tile % nty; tile /= nty;
  const int tz = tile % ntz;
  const int b = tile / ntz;
  const int x0 = tx * TX, y0 = ty * TY, z0 = tz * TZ;
  const int nz = min(TZ, w.out_n0 - z0);                 // every tile of the grid has at least one output
  if (threadIdx.x == 255) {
    mbar_init(bar, 1);
    fence_mbar_init();
    // box = [first corner of the tile's first output, last corner of its last output] per axis; x start aligned
    const int lz = resize_axis(g.S[0], w.M[0], w.delta[0], w.out_z0 + z0).i0;
    const int hz = resize_axis(g.S[0], w.M[0], w.delta[0], w.out_z0 + z0 + nz - 1).i1;
    const int ly = resize_axis(g.S[1], w.M[1], w.delta[1], y0).i0;
    const int hy = resize_axis(g.S[1], w.M[1], w.delta[1], min(y0 + TY, w.M[1]) - 1).i1;
    int lx = resize_axis(g.S[2], w.M[2], w.delta[2], x0).i0;
    const int hx = resize_axis(g.S[2], w.M[2], w.delta[2], min(x0 + TX, w.M[2]) - 1).i1;
    lx -= lx % xalign;
    const int ok = (hz - lz + 1 <= bxs.bz) && (hy - ly + 1 <= bxs.by) && (hx - lx + 1 <= bxs.bx) && !unstaged;
    s_lo[0] = lz; s_lo[1] = ly; s_lo[2] = lx; s_lo[3] = ok;
    if (ok) {
      mbar_expect_tx(bar, (uint32_t)(box_elems * sizeof(float)));
      tma_load_4d(s_box, &tm_vol, bar, lx * CT, ly, lz, b);
    }
  } else if (threadIdx.x < NT) {
    const int t = threadIdx.x;
    const int d = t < TZ ? 0 : (t < TZ + TY ? 1 : 2);
    const int i = d == 0 ? w.out_z0 + z0 + t : (d == 1 ? y0 + (t - TZ) : x0 + (t - TZ - TY));
    const int Sd = d == 0 ? g.S[0] : (d == 1 ? g.S[1] : g.S[2]);
    const int Md = d == 0 ? w.M[0] : (d == 1 ? w.M[1] : w.M[2]);
    const float dd = d == 0 ? w.delta[0] : (d == 1 ? w.delta[1] : w.delta[2]);
    float2 ww = make_float2(0.f, 0.f);
    int i0 = -1, i1 = -1;
    if (i < Md && (d != 0 || t < nz)) {
      const Axis a = resize_axis(Sd, Md, dd, i);
      i0 = a.i0; i1 = a.i1; ww = make_float2(a.wlo, a.whi);
    }
    s_w[t] = ww; s_i[0][t] = i0; s_i[1][t] = i1;
  }
  __syncthreads();
  const bool staged = s_lo[3] != 0;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int row = wid * 2 + (lane >> 4), xp = lane & 15;
  const int ox = x0 + 2 * xp, oy = y0 + row;
  if (staged) mbar_wait(bar, 0);
  if (oy >= w.M[1] || ox >= w.M[2]) return;
  const int zs = staged ? bxs.by * bxs.bx * CT : g.S[1] * g.S[2] * CT;
  const int ys = staged ? bxs.bx * CT : g.S[2] * CT;
  const int lz = staged ? s_lo[0] : 0, ly = staged ? s_lo[1] : 0, lx = staged ? s_lo[2] : 0;
  const bool has1 = ox + 1 < w.M[2];                    // odd output width: the pair's second voxel may not exist
  const int ta = TZ + TY + 2 * xp, tb = has1 ? ta + 1 : ta;     // (a missing second voxel repeats the first: legal reads)
  const float2 wy = s_w[TZ + row], wa = s_w[ta], wb = s_w[tb];
  const int y_o0 = (s_i[0][TZ + row] - ly) * ys, y_o1 = (s_i[1][TZ + row] - ly) * ys;
  const int a_o0 = (s_i[0][ta] - lx) * CT, a_o1 = (s_i[1][ta] - lx) * CT;
  const int b_o0 = (s_i[0][tb] - lx) * CT, b_o1 = (s_i[1][tb] - lx) * CT;
  const int oa[4] = {y_o0 + a_o0, y_o0 + a_o1, y_o1 + a_o0, y_o1 + a_o1};
  const int ob[4] = {y_o0 + b_o0, y_o0 + b_o1, y_o1 + b_o0, y_o1 + b_o1};
  float* outb = out + ((size_t)b * w.out_vox + ((size_t)z0 * w.M[1] + oy) * w.M[2] + ox) * CT;
  size_t plane = (size_t)w.M[1] * w.M[2] * CT;
  asm volatile("" : "+l"(plane));                       // opaque: keeps it in registers (it was re-derived from the parameters every plane)
  const f32x2 exlo = pack2(wa.x, wb.x), exhi = pack2(wa.y, wb.y);
  if (staged)
    resize_pair_march<CT, TZ, true>(smem_u32(s_box), nullptr, oa, ob, zs, lz, s_w, s_i[0], s_i[1], nz, wy, exlo, exhi,
                                    outb, plane, has1, negzero2, one2);
  else                                                  // box larger than the staged extents: straight from global memory
    resize_pair_march<CT, TZ, false>(0u, vol + (size_t)b * w.src_batch_stride, oa, ob, zs, lz, s_w, s_i[0], s_i[1], nz,
                                     wy, exlo, exhi, outb, plane, has1, negzero2, one2);
}

// largest source extent any tile of T outputs needs along one axis, with the device's fp32 linspace arithmetic
static int resize_axis_extent(int S, int M, float delta, int first, int count, int T, int align) {
  int ext = 1;
  for (int t0 = first; t0 < first + count; t0 += T) {
    const int t1 = (t0 + T - 1 < first + count - 1) ? t0 + T - 1 : first + count - 1;
    auto cell = [&](int i, int& i0, int& i1) {
      const float loc = (i == M - 1 && M > 1) ? (float)(S - 1) : delta * (float)i;
      float f0 = floorf(loc); f0 = f0 < 0.f ? 0.f : (f0 > (float)(S - 1) ? (float)(S - 1) : f0);
      float f1 = f0 + 1.0f; f1 = f1 > (float)(S - 1) ? (float)(S - 1) : f1;
      i0 = (int)f0; i1 = (int)f1;
    };
    int a0, a1, b0, b1;
    cell(t0, a0, a1); cell(t1, b0, b1);
    int lo = a0 - a0 % align;
    int hi = b1 > a1 ? b1 : a1;
    if (hi - lo + 1 > ext) ext = hi - lo + 1;
  }
  return ext;
}

// ---------------------------------------------------------------------------------------
// warp3d_tile_kernel: D=3, C=1, TMA-staged flow tile + source box in shared memory
// ---------------------------------------------------------------------------------------
struct TileGeo {
  Geo g;                 // S = {full_s0, H, W}
  int out_z0, out_n0;
  int B;
  int ntz, nty, ntx;     // tiles per axis
  int64_t src_batch_stride, out_vox;
  int64_t flow_bstride, out_bstride;   // elements between batch items of flow / out
  int abs_loc;           // 1: the 'flow' tensor holds absolute sample locations (interpn on the volume's own grid)
};

// Compile-time tile / box geometry.  HZ = HY = HALO; the x halo is rounded up to 4 voxels
// because the TMA needs the innermost start coordinate 16-byte aligned.
// CC = channels staged per voxel (1..4): the box keeps the volume's channels-last layout, so
// (x, c) is one contiguous TMA dimension of BX*CC floats.
template <int TZ, int TY, int HALO, int CC = 1>
struct TileCfg {
  static constexpr int TX = 32, NW = 8;
  static constexpr int HX = (HALO + 3) & ~3;
  static constexpr int BZ = TZ + 2 * HALO, BY = TY + 2 * HALO, BX = TX + 2 * HX;
  static constexpr int ROWS = TY / NW;                  // rows of 32 voxels per warp per plane
  static constexpr int FLOW_ELEMS = TZ * TY * TX * 3, BOX_ELEMS = BZ * BY * BX * CC;
  static_assert(BX * CC <= 256, "TMA box limit on the merged (x, channel) dimension");
  static constexpr size_t SMEM = (size_t)(FLOW_ELEMS + BOX_ELEMS) * sizeof(float) + 32;   // + 2 mbarriers + box origin
  static_assert(TY % NW == 0, "TY must be a multiple of the warp count");
  static_assert(BX <= 256 && BY <= 256 && BZ <= 256, "TMA box limit");
};

// the 8 corner products and the accumulation, in the reference's order (utils.py:159-191)
__device__ __forceinline__ float trilerp(const float (&v)[8], float wz0, float wz1, float wy0, float wy1,
                                         float wx0, float wx1) {
  const float w00 = __fmul_rn(wz0, wy0), w01 = __fmul_rn(wz0, wy1);
  const float w10 = __fmul_rn(wz1, wy0), w11 = __fmul_rn(wz1, wy1);
  float r = __fadd_rn(0.f, __fmul_rn(__fmul_rn(w00, wx0), v[0]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w00, wx1), v[1]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w01, wx0), v[2]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w01, wx1), v[3]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w10, wx0), v[4]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w10, wx1), v[5]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w11, wx0), v[6]));
  r = __fadd_rn(r, __fmul_rn(__fmul_rn(w11, wx1), v[7]));
  return r;
}


// CC channels of one voxel, as one vector store where the alignment allows it
template <int CC>
__device__ __forceinline__ void store_channels(float* __restrict__ op, const float (&res)[CC]) {
  if (CC == 4) {
    *reinterpret_cast<float4*>(op) = make_float4(res[0], res[1 % CC], res[2 % CC], res[3 % CC]);
  } else if (CC == 2) {
    *reinterpret_cast<float2*>(op) = make_float2(res[0], res[1 % CC]);
  } else {
#pragma unroll
    for (int c = 0; c < CC; ++c) op[c] = res[c];
  }
}

// general (any position, any flow) sample through global memory -- the semantics baseline
template <int METHOD, int CC = 1>
__device__ __forceinline__ void sample_global3(const float* __restrict__ volb, const Geo& g,
                                               float lz, float ly, float lx, float (&res)[CC]) {
  if (METHOD == NRT_LINEAR) {
    Axis az = axis_linear(lz, (float)(g.S[0] - 1), g.S[0] - 1);
    const Axis ay = axis_linear(ly, (float)(g.S[1] - 1), g.S[1] - 1);
    const Axis ax = axis_linear(lx, (float)(g.S[2] - 1), g.S[2] - 1);
    az.i0 = to_resident(g, az.i0);
    az.i1 = to_resident(g, az.i1);
    const int r00 = (az.i0 * g.S[1] + ay.i0) * g.S[2], r01 = (az.i0 * g.S[1] + ay.i1) * g.S[2];
    const int r10 = (az.i1 * g.S[1] + ay.i0) * g.S[2], r11 = (az.i1 * g.S[1] + ay.i1) * g.S[2];
    const int idx[8] = {r00 + ax.i0, r00 + ax.i1, r01 + ax.i0, r01 + ax.i1, r10 + ax.i0, r10 + ax.i1, r11 + ax.i0, r11 + ax.i1};
    float k[8];
    corner_weights(az.wlo, az.whi, ay.wlo, ay.whi, ax.wlo, ax.whi, k);
#pragma unroll
    for (int c = 0; c < CC; ++c) {
      float v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = __ldg(volb + (size_t)idx[q] * CC + c);
      res[c] = acc8(k, v);
    }
  } else {
    const int iz = to_resident(g, axis_nearest(lz, g.S[0] - 1));
    const int iy = axis_nearest(ly, g.S[1] - 1), ix = axis_nearest(lx, g.S[2] - 1);
#pragma unroll
    for (int c = 0; c < CC; ++c) res[c] = __ldg(volb + (size_t)((iz * g.S[1] + iy) * g.S[2] + ix) * CC + c);
  }
}


// The rows of one staged tile owned by this warp.  Branch-free main loop: a voxel whose
// corners are not all inside the staged box still runs the shared-memory arithmetic on a
// clamped (legal, meaningless) address; the thread only remembers THAT it happened (one
// predicate for all its voxels) and re-checks its voxels after the loop, recomputing the
// affected ones through global memory.  Without a divergent branch or mask bookkeeping in the
// body the compiler can overlap the LDS latency of one iteration with the multiply/add chain
// of the previous one.
//   GENERAL = true : run-time `partial` (tile overhangs the output) and `has_fill` handling
//   GENERAL = false: full tile, no fill value -- neither test exists in the loop
template <int TZ, int TY, int HALO, int METHOD, bool EZ, bool EY, bool EX, int CC, bool ABS, bool GENERAL>
__device__ __forceinline__ void tile_rows(const float* __restrict__ s_flow, const float* __restrict__ s_box,
                                          const float* __restrict__ volb, float* __restrict__ outb,
                                          const TileGeo& w, int x0, int y0, int z0l, int ox, int oy, int oz,
                                          bool partial_rt) {
  using Cfg = TileCfg<TZ, TY, HALO, CC>;
  constexpr int TX = Cfg::TX, BX = Cfg::BX, BY = Cfg::BY, BZ = Cfg::BZ, NW = Cfg::NW;
  constexpr int ZSTEP = NW >= TY ? NW / TY : 1;          // planes between a warp's rows
  constexpr int YROWS = NW >= TY ? 1 : TY / NW;          // rows per plane per warp
  const Geo& g = w.g;
  const int H = g.S[1], W = g.S[2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int zs = NW >= TY ? wid / TY : 0;
  const int gz0 = w.out_z0 + z0l;
  const int gx = x0 + lane;
  const bool partial = GENERAL && partial_rt;
  const bool has_fill = GENERAL && g.has_fill;
  // with absolute locations the grid term is 0 (0 + x == x exactly): same instruction count
  const float fx = ABS ? 0.f : (float)gx;
  BoxBounds bb;
  bb.lo_z = max(oz, g.src_z0); bb.hi_z = min(oz + BZ - 1, g.src_z0 + g.src_n0 - 1);
  bb.lo_y = max(oy, 0); bb.hi_y = min(oy + BY - 1, H - 1);
  bb.lo_x = max(ox, 0); bb.hi_x = min(ox + BX - 1, W - 1);
  const int nz_out = partial ? min(TZ, w.out_n0 - z0l) : TZ;
#pragma unroll
  for (int yr = 0; yr < YROWS; ++yr) {
    const int yy = (NW >= TY ? wid % TY : wid) + yr * NW;
    const int gy = y0 + yy;
    if (partial && (gx >= W || gy >= H)) continue;
    const float fy = ABS ? 0.f : (float)gy;
    float zf = ABS ? 0.f : (float)(gz0 + zs);                 // running z coordinate (exact small integers)
    const float zstep = ABS ? 0.f : (float)ZSTEP;
    const float* fl = s_flow + ((zs * TY + yy) * TX + lane) * 3;
    float* op = outb + (((size_t)(z0l + zs) * H + gy) * W + gx) * CC;
    bool all_ok = true;
    const float* fl0 = fl;
    float* op0 = op;
#pragma unroll 2
    for (int z = zs; z < TZ; z += ZSTEP, fl += ZSTEP * TY * TX * 3, op += (size_t)ZSTEP * H * W * CC, zf += zstep) {
      if (partial && z >= nz_out) break;
      const float lz = __fadd_rn(zf, fl[0]);
      const float ly = __fadd_rn(fy, fl[1]);
      const float lx = __fadd_rn(fx, fl[2]);
      float res[CC];
      if (METHOD == NRT_LINEAR) {
        AxisBox<EZ, BZ> az; AxisBox<EY, BY> ay; AxisBox<EX, BX> ax;
        az.setup(lz, oz, bb.lo_z, bb.hi_z, g.S[0] - 1);
        ay.setup(ly, oy, bb.lo_y, bb.hi_y, H - 1);
        ax.setup(lx, ox, bb.lo_x, bb.hi_x, W - 1);
        const float* p = s_box + ((az.c0 * BY + ay.c0) * BX + ax.c0) * CC;
        const int dz = (EZ ? az.d * (BY * BX) : BY * BX) * CC;
        const int dy = (EY ? ay.d * BX : BX) * CC;
        const int dx = (EX ? ax.d : 1) * CC;
        if (CC == 1) {
          float v[8];
          v[0] = p[0];       v[1] = p[dx];
          v[2] = p[dy];      v[3] = p[dy + dx];
          v[4] = p[dz];      v[5] = p[dz + dx];
          v[6] = p[dz + dy]; v[7] = p[dz + dy + dx];
          res[0] = trilerp(v, az.wlo, az.whi, ay.wlo, ay.whi, ax.wlo, ax.whi);
        } else {
          float k[8];
          corner_weights(az.wlo, az.whi, ay.wlo, ay.whi, ax.wlo, ax.whi, k);
          const int off[8] = {0, dx, dy, dy + dx, dz, dz + dx, dz + dy, dz + dy + dx};
#pragma unroll
          for (int c = 0; c < CC; ++c) {
            float v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = p[off[q] + c];
            res[c] = acc8(k, v);
          }
        }
        all_ok = all_ok & az.ok & ay.ok & ax.ok;
      } else {
        bool ok = true;
        const int cz = nearest_box<EZ, BZ>(lz, oz, bb.lo_z, bb.hi_z, g.S[0] - 1, ok);
        const int cy = nearest_box<EY, BY>(ly, oy, bb.lo_y, bb.hi_y, H - 1, ok);
        const int cx = nearest_box<EX, BX>(lx, ox, bb.lo_x, bb.hi_x, W - 1, ok);
#pragma unroll
        for (int c = 0; c < CC; ++c) res[c] = s_box[((cz * BY + cy) * BX + cx) * CC + c];
        all_ok = all_ok & ok;
      }
      if (has_fill) {
#pragma unroll
        for (int c = 0; c < CC; ++c) res[c] = fill_if_oob(g, res[c], lz, ly, lx);
      }
      store_channels<CC>(op, res);
    }
    if (!all_ok) {                                     // rare: some corner of some voxel outside the staged box
#pragma unroll 1
      for (int z = zs, it = 0; z < nz_out; z += ZSTEP, ++it) {
        const float* f2 = fl0 + (size_t)it * ZSTEP * TY * TX * 3;
        const float lz = __fadd_rn(ABS ? 0.f : (float)(gz0 + z), f2[0]);
        const float ly = __fadd_rn(fy, f2[1]);
        const float lx = __fadd_rn(fx, f2[2]);
        bool ok = true;
        if (METHOD == NRT_LINEAR) {
          AxisBox<EZ, BZ> az; AxisBox<EY, BY> ay; AxisBox<EX, BX> ax;           // the very test of the main loop
          az.setup(lz, oz, bb.lo_z, bb.hi_z, g.S[0] - 1);
          ay.setup(ly, oy, bb.lo_y, bb.hi_y, H - 1);
          ax.setup(lx, ox, bb.lo_x, bb.hi_x, W - 1);
          ok = az.ok & ay.ok & ax.ok;
        } else {
          (void)nearest_box<EZ, BZ>(lz, oz, bb.lo_z, bb.hi_z, g.S[0] - 1, ok);
          (void)nearest_box<EY, BY>(ly, oy, bb.lo_y, bb.hi_y, H - 1, ok);
          (void)nearest_box<EX, BX>(lx, ox, bb.lo_x, bb.hi_x, W - 1, ok);
        }
        if (ok) continue;                              // this one was computed from the box: keep it
        float res[CC];
        sample_global3<METHOD, CC>(volb, g, lz, ly, lx, res);
        if (g.has_fill) {
#pragma unroll
          for (int c = 0; c < CC; ++c) res[c] = fill_if_oob(g, res[c], lz, ly, lx);
        }
        store_channels<CC>(op0 + (size_t)it * ZSTEP * H * W * CC, res);
      }
    }
  }
}

// Process one staged tile.  Warp w owns row y = w % TY of planes z = w / TY, + NW/TY, ...
// The per-axis EDGE flags are tile-uniform, so the dispatch below costs one uniform switch.  Tiles that overhang
// the output and launches with a fill value take the one general variant (all edges, run-time checks).
template <int TZ, int TY, int HALO, int METHOD, int CC = 1, bool ABS = false>
__device__ __forceinline__ void compute_tile(const float* __restrict__ s_flow, const float* __restrict__ s_box,
                                             const float* __restrict__ volb, float* __restrict__ outb,
                                             const TileGeo& w, int x0, int y0, int z0l, int ox, int oy, int oz) {
  using Cfg = TileCfg<TZ, TY, HALO, CC>;
  const Geo& g = w.g;
  const bool ez = !((oz >= g.src_z0) && (oz + Cfg::BZ <= g.src_z0 + g.src_n0));
  const bool ey = !((oy >= 0) && (oy + Cfg::BY <= g.S[1]));
  const bool ex = !((ox >= 0) && (ox + Cfg::BX <= g.S[2]));
  const bool partial = (z0l + TZ > w.out_n0) || (y0 + TY > g.S[1]) || (x0 + Cfg::TX > g.S[2]);
#define NRT_ROWS(a, b, c, gen) tile_rows<TZ, TY, HALO, METHOD, a, b, c, CC, ABS, gen>(s_flow, s_box, volb, outb, w, x0, y0, z0l, ox, oy, oz, partial)
  if (partial || g.has_fill) { NRT_ROWS(true, true, true, true); return; }
  switch ((ez ? 4 : 0) | (ey ? 2 : 0) | (ex ? 1 : 0)) {
    case 0: NRT_ROWS(false, false, false, false); break;
    case 1: NRT_ROWS(false, false, true, false); break;
    case 2: NRT_ROWS(false, true, false, false); break;
    case 3: NRT_ROWS(false, true, true, false); break;
    case 4: NRT_ROWS(true, false, false, false); break;
    case 5: NRT_ROWS(true, false, true, false); break;
    case 6: NRT_ROWS(true, true, false, false); break;
    default: NRT_ROWS(true, true, true, false); break;
  }
#undef NRT_ROWS
}

// v1: one tile per CTA, several CTAs per SM overlap each other's load phase.  3-D grid
// (x tiles, y tiles, z tiles * batch) keeps the per-CTA prologue free of div/mod chains:
// with only 8-16 voxels per thread the prologue is a visible part of the instruction count.
// ABS = the 'flow' tensor holds absolute sample locations (interpn on the volume's own grid): compile-time, so
// that the displacement kernels carry no trace of it
template <int TZ, int TY, int HALO, int METHOD, int CC = 1, bool ABS = false>
__global__ void __launch_bounds__(TileCfg<TZ, TY, HALO, CC>::NW * 32)
warp3d_tile_kernel(const __grid_constant__ CUtensorMap tm_vol,
                   const __grid_constant__ CUtensorMap tm_flow,
                   const float* __restrict__ vol, float* __restrict__ out, TileGeo w, int follow) {
  using Cfg = TileCfg<TZ, TY, HALO, CC>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_flow = reinterpret_cast<float*>(smem_raw);                       // [TZ][TY][TX][3]
  float* s_box = s_flow + Cfg::FLOW_ELEMS;                                  // [BZ][BY][BX]
  uint64_t* bar = reinterpret_cast<uint64_t*>(s_box + Cfg::BOX_ELEMS);     // bar[0]: source box, bar[1]: flow tile
  int* s_org = reinterpret_cast<int*>(bar + 2);                             // mean shift of the tile (box re-staging)
  const int b = blockIdx.z / w.ntz;
  const int x0 = blockIdx.x * Cfg::TX, y0 = blockIdx.y * TY, z0l = (blockIdx.z - b * w.ntz) * TZ;
  if (threadIdx.x == 0) {
    // speculative load: flow tile + the box centred on the tile itself (right for small or
    // incoherent displacements), issued before anything is known about the flow.  The flow tile goes first and on
    // its own barrier: the warp that inspects it can start while the (larger) box is still landing.
    mbar_init(bar, 1);
    mbar_init(bar + 1, 1);
    fence_mbar_init();
    mbar_expect_tx(bar + 1, (uint32_t)(Cfg::FLOW_ELEMS * sizeof(float)));
    tma_load_4d(s_flow, &tm_flow, bar + 1, x0 * 3, y0, z0l, b);
    mbar_expect_tx(bar, (uint32_t)(Cfg::BOX_ELEMS * sizeof(float)));
    tma_load_4d(s_box, &tm_vol, bar, (x0 - Cfg::HX) * CC, y0 - HALO, w.out_z0 + z0l - HALO - w.g.src_z0, b);
  }
  __syncthreads();                                   // the barriers are initialised
  mbar_wait(bar + 1, 0);
  // Where does the tile land ON AVERAGE?  ONE warp looks at a 3x3x3 lattice of the STAGED flow tile (27 lanes, one
  // LDS per component: no global latency) and sums the shifts in 1/64-voxel fixed point with the warp-reduce
  // instruction (three REDUX instead of fifteen shuffle + add steps).  A large coherent displacement means the
  // speculative box is useless; the box is then re-staged around the displaced position, so that the halo only has
  // to cover the variation of the flow inside the tile.  An incoherent flow averages out and keeps the box.
  // (Every warp doing this redundantly would add 8 x 60 instructions per tile, ~9 % of the tile's instruction count;
  // one warp + one block barrier is far cheaper.)
  int sz = 0, sy = 0, sx = 0;
  if (follow) {                                      // launch-uniform
    if (threadIdx.x < 32) {
      int mz = 0, my = 0, mx = 0;
      const int l = threadIdx.x;
      if (l < 27) {
        const int jz = l / 9, jy = (l / 3) % 3, jx = l % 3;
        const int cz = min(z0l + (jz * (TZ - 1)) / 2, w.out_n0 - 1);
        const int cy = min(y0 + (jy * (TY - 1)) / 2, w.g.S[1] - 1);
        const int cx = min(x0 + (jx * (Cfg::TX - 1)) / 2, w.g.S[2] - 1);
        const float* f = s_flow + (((cz - z0l) * TY + (cy - y0)) * Cfg::TX + (cx - x0)) * 3;
        const float lim = 16384.f;                   // |shift| beyond this is clamped: 27 * 64 * 16384 < 2^31
        const float gz_ = ABS ? (float)(w.out_z0 + cz) : 0.f, gy_ = ABS ? (float)cy : 0.f, gx_ = ABS ? (float)cx : 0.f;
        mz = __float2int_rn(fminf(fmaxf(f[0] - gz_, -lim), lim) * 64.f);
        my = __float2int_rn(fminf(fmaxf(f[1] - gy_, -lim), lim) * 64.f);
        mx = __float2int_rn(fminf(fmaxf(f[2] - gx_, -lim), lim) * 64.f);
      }
      mz = __reduce_add_sync(0xffffffffu, mz); my = __reduce_add_sync(0xffffffffu, my); mx = __reduce_add_sync(0xffffffffu, mx);
      // dead band: 2 voxels in z/y, 4 in x (the TMA needs the x start 16-byte aligned and the x halo is already
      // rounded up to 4); thresholds in units of 1/64 voxel summed over 27 samples
      int3 s = make_int3(0, 0, 0);
      if (abs(mz) >= 2 * 64 * 27 || abs(my) >= 2 * 64 * 27 || abs(mx) >= 4 * 64 * 27) {
        s.z = __float2int_rn((float)mz * (1.f / (64.f * 27.f)));
        s.y = __float2int_rn((float)my * (1.f / (64.f * 27.f)));
        s.x = __float2int_rn((float)mx * (1.f / (64.f * 27.f * 4.f))) * 4;
      }
      if (threadIdx.x == 0) { s_org[0] = s.z; s_org[1] = s.y; s_org[2] = s.x; }
    }
    __syncthreads();
    sz = s_org[0]; sy = s_org[1]; sx = s_org[2];
  }
  mbar_wait(bar, 0);
  const int oz = w.out_z0 + z0l - HALO + sz, oy = y0 - HALO + sy, ox = x0 - Cfg::HX + sx;
  if ((sz | sy | sx) != 0) {                         // block-uniform
    // every thread must have observed phase 0 before phase 1 is armed: an mbarrier waiter
    // can be at most one phase behind (parity aliasing), found with compute-sanitizer
    __syncthreads();
    if (threadIdx.x == 0) {
      mbar_expect_tx(bar, (uint32_t)(Cfg::BOX_ELEMS * sizeof(float)));
      tma_load_4d(s_box, &tm_vol, bar, ox * CC, oy, oz - w.g.src_z0, b);
    }
    mbar_wait(bar, 1);
  }
  compute_tile<TZ, TY, HALO, METHOD, CC, ABS>(s_flow, s_box, vol + (size_t)b * w.src_batch_stride,
                                         out + (size_t)b * w.out_bstride, w, x0, y0, z0l, ox, oy, oz);
}

// ---------------------------------------------------------------------------------------
// warp3d_bwd_tile_kernel: gradient of the D=3, C=1 warp.  Same staging as the forward
// (flow tile + source box by TMA, plus the upstream-gradient tile); d/dvol is accumulated
// into a shared-memory box with shared atomics and flushed once per tile with 128-bit
// vector reductions (red.global.add.v4.f32), i.e. ~1 global atomic per output voxel
// instead of 8; d/dflow is written directly.  Voxels whose corners fall outside the
// staged box go straight to global memory.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// d out / d loc for one sample, given corner values v (order 000..111) and the per-axis weights
__device__ __forceinline__ void trilerp_grad(const float (&v)[8], float wz0, float wz1, float wy0, float wy1,
                                             float wx0, float wx1, float& gz, float& gy, float& gx) {
  // corner bit 0 carries weight w0 = f1 - x (d/dx = -1), bit 1 carries w1 = 1 - w0 (d/dx = +1)
  gx = wz0 * (wy0 * (v[1] - v[0]) + wy1 * (v[3] - v[2])) + wz1 * (wy0 * (v[5] - v[4]) + wy1 * (v[7] - v[6]));
  gy = wz0 * (wx0 * (v[2] - v[0]) + wx1 * (v[3] - v[1])) + wz1 * (wx0 * (v[6] - v[4]) + wx1 * (v[7] - v[5]));
  gz = wy0 * (wx0 * (v[4] - v[0]) + wx1 * (v[5] - v[1])) + wy1 * (wx0 * (v[6] - v[2]) + wx1 * (v[7] - v[3]));
}

template <int METHOD>
__device__ __forceinline__ void bwd_global3(const float* __restrict__ volb, float* __restrict__ gvolb, const Geo& g,
                                            float lz, float ly, float lx, float go, bool want_flow,
                                            float& gz, float& gy, float& gx) {
  gz = gy = gx = 0.f;
  if (METHOD == NRT_LINEAR) {
    const Axis az = axis_linear(lz, (float)(g.S[0] - 1), g.S[0] - 1);
    const Axis ay = axis_linear(ly, (float)(g.S[1] - 1), g.S[1] - 1);
    const Axis ax = axis_linear(lx, (float)(g.S[2] - 1), g.S[2] - 1);
    const int r00 = (az.i0 * g.S[1] + ay.i0) * g.S[2], r01 = (az.i0 * g.S[1] + ay.i1) * g.S[2];
    const int r10 = (az.i1 * g.S[1] + ay.i0) * g.S[2], r11 = (az.i1 * g.S[1] + ay.i1) * g.S[2];
    const int idx[8] = {r00 + ax.i0, r00 + ax.i1, r01 + ax.i0, r01 + ax.i1, r10 + ax.i0, r10 + ax.i1, r11 + ax.i0, r11 + ax.i1};
    const float w[8] = {az.wlo * ay.wlo * ax.wlo, az.wlo * ay.wlo * ax.whi, az.wlo * ay.whi * ax.wlo, az.wlo * ay.whi * ax.whi,
                        az.whi * ay.wlo * ax.wlo, az.whi * ay.wlo * ax.whi, az.whi * ay.whi * ax.wlo, az.whi * ay.whi * ax.whi};
    float v[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      if (gvolb) atomicAdd(gvolb + idx[c], w[c] * go);
      v[c] = want_flow ? __ldg(volb + idx[c]) : 0.f;
    }
    if (want_flow) {
      trilerp_grad(v, az.wlo, az.whi, ay.wlo, ay.whi, ax.wlo, ax.whi, gz, gy, gx);
      gz = (lz >= 0.f && lz <= (float)(g.S[0] - 1)) ? gz * go : 0.f;
      gy = (ly >= 0.f && ly <= (float)(g.S[1] - 1)) ? gy * go : 0.f;
      gx = (lx >= 0.f && lx <= (float)(g.S[2] - 1)) ? gx * go : 0.f;
    }
  } else if (gvolb) {
    const int iz = axis_nearest(lz, g.S[0] - 1), iy = axis_nearest(ly, g.S[1] - 1), ix = axis_nearest(lx, g.S[2] - 1);
    atomicAdd(gvolb + (iz * g.S[1] + iy) * g.S[2] + ix, go);
  }
}

template <int METHOD>
__global__ void __launch_bounds__(256)
warp3d_bwd_tile_kernel(const __grid_constant__ CUtensorMap tm_vol, const __grid_constant__ CUtensorMap tm_flow,
                       const __grid_constant__ CUtensorMap tm_gout, const float* __restrict__ vol,
                       float* __restrict__ gvol, float* __restrict__ gflow, TileGeo w) {
  constexpr int TZ = 8, TY = 8, HALO = 3, NW = 8;
  using Cfg = TileCfg<TZ, TY, HALO>;
  constexpr int TX = Cfg::TX, BX = Cfg::BX, BY = Cfg::BY, BZ = Cfg::BZ;
  constexpr int GOUT_ELEMS = TZ * TY * TX;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_flow = reinterpret_cast<float*>(smem_raw);                       // [TZ][TY][TX][3]
  float* s_box = s_flow + Cfg::FLOW_ELEMS;                                  // [BZ][BY][BX] source values
  float* s_gout = s_box + Cfg::BOX_ELEMS;                                   // [TZ][TY][TX]
  float* s_acc = s_gout + GOUT_ELEMS;                                       // [BZ][BY][BX] d/dvol accumulator
  uint64_t* bar = reinterpret_cast<uint64_t*>(s_acc + Cfg::BOX_ELEMS);
  const Geo& g = w.g;
  const int H = g.S[1], W = g.S[2];
  const int b = blockIdx.z / w.ntz;
  const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY, z0 = (blockIdx.z - b * w.ntz) * TZ;
  const int ox = x0 - Cfg::HX, oy = y0 - HALO, oz = z0 - HALO;
  const bool want_flow = gflow != nullptr && METHOD == NRT_LINEAR;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    mbar_expect_tx(bar, (uint32_t)((Cfg::FLOW_ELEMS + Cfg::BOX_ELEMS + GOUT_ELEMS) * sizeof(float)));
    tma_load_4d(s_flow, &tm_flow, bar, x0 * 3, y0, z0, b);
    tma_load_4d(s_box, &tm_vol, bar, ox, oy, oz, b);
    tma_load_4d(s_gout, &tm_gout, bar, x0, y0, z0, b);
  }
  for (int i = threadIdx.x; i < Cfg::BOX_ELEMS; i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  mbar_wait(bar, 0);

  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int gx_ = x0 + lane, gy_ = y0 + wid;
  const float* volb = vol + (size_t)b * w.src_batch_stride;
  float* gvolb = gvol ? gvol + (size_t)b * w.src_batch_stride : nullptr;
  BoxBounds bb;
  bb.lo_z = max(oz, 0); bb.hi_z = min(oz + BZ - 1, g.S[0] - 1);
  bb.lo_y = max(oy, 0); bb.hi_y = min(oy + BY - 1, H - 1);
  bb.lo_x = max(ox, 0); bb.hi_x = min(ox + BX - 1, W - 1);
  if (gx_ < W && gy_ < H) {
    for (int z = 0; z < TZ && z0 + z < g.S[0]; ++z) {
      const int t = (z * TY + wid) * TX + lane;
      const float go = s_gout[t];
      const float lz = __fadd_rn((float)(z0 + z), s_flow[t * 3 + 0]);
      const float ly = __fadd_rn((float)gy_, s_flow[t * 3 + 1]);
      const float lx = __fadd_rn((float)gx_, s_flow[t * 3 + 2]);
      float gz = 0.f, gy = 0.f, gx = 0.f;
      const bool oob = g.has_fill && ((lz < 0.f) | (lz > (float)(g.S[0] - 1)) | (ly < 0.f) | (ly > (float)(H - 1)) |
                                      (lx < 0.f) | (lx > (float)(W - 1)));
      if (!oob) {
        if (METHOD == NRT_LINEAR) {
          AxisBox<true, BZ> az; AxisBox<true, BY> ay; AxisBox<true, BX> ax;
          az.setup(lz, oz, bb.lo_z, bb.hi_z, g.S[0] - 1);
          ay.setup(ly, oy, bb.lo_y, bb.hi_y, H - 1);
          ax.setup(lx, ox, bb.lo_x, bb.hi_x, W - 1);
          if (az.ok & ay.ok & ax.ok) {
            const int base = (az.c0 * BY + ay.c0) * BX + ax.c0;
            const int dz = az.d * (BY * BX), dy = ay.d * BX, dx = ax.d;
            const int off[8] = {0, dx, dy, dy + dx, dz, dz + dx, dz + dy, dz + dy + dx};
            const float w00 = az.wlo * ay.wlo, w01 = az.wlo * ay.whi, w10 = az.whi * ay.wlo, w11 = az.whi * ay.whi;
            const float wc[8] = {w00 * ax.wlo, w00 * ax.whi, w01 * ax.wlo, w01 * ax.whi,
                                 w10 * ax.wlo, w10 * ax.whi, w11 * ax.wlo, w11 * ax.whi};
            float v[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              if (gvolb) atomicAdd(s_acc + base + off[c], wc[c] * go);
              v[c] = s_box[base + off[c]];
            }
            if (want_flow) {
              trilerp_grad(v, az.wlo, az.whi, ay.wlo, ay.whi, ax.wlo, ax.whi, gz, gy, gx);
              gz = (lz >= 0.f && lz <= (float)(g.S[0] - 1)) ? gz * go : 0.f;
              gy = (ly >= 0.f && ly <= (float)(H - 1)) ? gy * go : 0.f;
              gx = (lx >= 0.f && lx <= (float)(W - 1)) ? gx * go : 0.f;
            }
          } else {
            bwd_global3<METHOD>(volb, gvolb, g, lz, ly, lx, go, want_flow, gz, gy, gx);
          }
        } else {
          const int iz = axis_nearest(lz, g.S[0] - 1), iy = axis_nearest(ly, H - 1), ix = axis_nearest(lx, W - 1);
          if ((iz >= bb.lo_z) & (iz <= bb.hi_z) & (iy >= bb.lo_y) & (iy <= bb.hi_y) & (ix >= bb.lo_x) & (ix <= bb.hi_x)) {
            if (gvolb) atomicAdd(s_acc + ((iz - oz) * BY + (iy - oy)) * BX + (ix - ox), go);
          } else {
            bwd_global3<METHOD>(volb, gvolb, g, lz, ly, lx, go, false, gz, gy, gx);
          }
        }
      }
      if (want_flow) {
        float* gf = gflow + ((((size_t)b * g.S[0] + (z0 + z)) * H + gy_) * W + gx_) * 3;
        gf[0] = gz; gf[1] = gy; gf[2] = gx;
      }
    }
  }
  if (!gvolb) return;
  __syncthreads();
  // flush the accumulator box: rows of BX floats, 4 at a time (ox and W are multiples of 4,
  // so every in-volume quad is 16-byte aligned and entirely inside or outside the volume)
  constexpr int QX = BX / 4;
  for (int q = threadIdx.x; q < BZ * BY * QX; q += blockDim.x) {
    const int qx = q % QX, r = q / QX;
    const int by_ = r % BY, bz_ = r / BY;
    const int gz_ = oz + bz_, gyy = oy + by_, gxx = ox + qx * 4;
    if (gz_ < 0 || gz_ >= g.S[0] || gyy < 0 || gyy >= H || gxx < 0 || gxx >= W) continue;
    const float4 a = *reinterpret_cast<const float4*>(s_acc + (bz_ * BY + by_) * BX + qx * 4);
    if (a.x == 0.f && a.y == 0.f && a.z == 0.f && a.w == 0.f) continue;
    red_add_v4(gvolb + ((size_t)gz_ * H + gyy) * W + gxx, a.x, a.y, a.z, a.w);
  }
}

// ---------------------------------------------------------------------------------------
// host: tensor-map encoding through the runtime's driver entry point (no -lcuda needed)
// ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    (void)cudaGetLastError();
  }
  return fn;
}

int encode_f32_tiled(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint32_t* box,
                     uint64_t last_stride_elems) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error(NRT_E_NODEV, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bx[5], es[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; }
  gstr[0] = dims[0] * sizeof(float);
  for (int i = 1; i < rank - 1; ++i) gstr[i] = gstr[i - 1] * dims[i];
  if (last_stride_elems) gstr[rank - 2] = last_stride_elems * sizeof(float);     // batch items not densely packed
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(NRT_E_LAUNCH, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
  return NRT_OK;
}

static int encode_f32_4d(CUtensorMap* tm, const void* base, const uint64_t dims[4], const uint32_t box[4],
                         uint64_t batch_stride_elems = 0) {
  return encode_f32_tiled(tm, base, 4, dims, box, batch_stride_elems);
}

int warp3d_bwd_tile(const float* vol, const float* flow, const float* gout, float* gvol, float* gflow, int B,
                    const int32_t* shape, int method, int has_fill, cudaStream_t st, bool* used) {
  *used = false;
  constexpr int TZ = 8, TY = 8, HALO = 3;
  using Cfg = TileCfg<TZ, TY, HALO>;
  const int D0 = shape[0], H = shape[1], W = shape[2];
  if (env_int("NRT_WARP_BWD_TILE", 1) == 0) return NRT_OK;
  if (W % 4 != 0 || W < 32 || !aligned16(vol) || !aligned16(flow) || !aligned16(gout) || (gvol && !aligned16(gvol)))
    return NRT_OK;
  TileGeo tg;
  tg.g.S[0] = D0; tg.g.S[1] = H; tg.g.S[2] = W;
  tg.g.src_z0 = 0; tg.g.src_n0 = D0; tg.g.C = 1; tg.g.has_fill = has_fill; tg.g.fill = 0.f; tg.g.err = nullptr;
  tg.out_z0 = 0; tg.out_n0 = D0; tg.B = B; tg.abs_loc = 0;
  tg.ntz = (D0 + TZ - 1) / TZ; tg.nty = (H + TY - 1) / TY; tg.ntx = (W + Cfg::TX - 1) / Cfg::TX;
  tg.src_batch_stride = (int64_t)D0 * H * W; tg.out_vox = tg.src_batch_stride;
  tg.flow_bstride = tg.out_vox * 3; tg.out_bstride = tg.out_vox;
  if ((int64_t)B * tg.ntz > 65535 || tg.nty > 65535) return NRT_OK;
  constexpr size_t SMEM = (size_t)(Cfg::FLOW_ELEMS + 2 * Cfg::BOX_ELEMS + TZ * TY * Cfg::TX) * sizeof(float) + 16;
  CUtensorMap tmv, tmf, tmg;
  const uint64_t vd[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)D0, (uint64_t)B};
  const uint32_t vb[4] = {(uint32_t)Cfg::BX, (uint32_t)Cfg::BY, (uint32_t)Cfg::BZ, 1};
  const uint64_t fd[4] = {(uint64_t)W * 3, (uint64_t)H, (uint64_t)D0, (uint64_t)B};
  const uint32_t fb[4] = {(uint32_t)Cfg::TX * 3, (uint32_t)TY, (uint32_t)TZ, 1};
  const uint32_t gb[4] = {(uint32_t)Cfg::TX, (uint32_t)TY, (uint32_t)TZ, 1};
  int rc = encode_f32_4d(&tmv, vol, vd, vb);
  if (rc == NRT_OK) rc = encode_f32_4d(&tmf, flow, fd, fb);
  if (rc == NRT_OK) rc = encode_f32_4d(&tmg, gout, vd, gb);
  if (rc != NRT_OK) return rc;
  const dim3 grid(tg.ntx, tg.nty, tg.ntz * B);
  *used = true;
  if (method == NRT_LINEAR) {
    // (set on every launch: the attribute is per device, and the call costs ~1 us)
    if (cudaFuncSetAttribute(warp3d_bwd_tile_kernel<NRT_LINEAR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess)
      return check_launch("cudaFuncSetAttribute(warp3d_bwd_tile)");
    warp3d_bwd_tile_kernel<NRT_LINEAR><<<grid, 256, SMEM, st>>>(tmv, tmf, tmg, vol, gvol, gflow, tg);
  } else {
    if (cudaFuncSetAttribute(warp3d_bwd_tile_kernel<NRT_NEAREST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM) != cudaSuccess)
      return check_launch("cudaFuncSetAttribute(warp3d_bwd_tile)");
    warp3d_bwd_tile_kernel<NRT_NEAREST><<<grid, 256, SMEM, st>>>(tmv, tmf, tmg, vol, gvol, gflow, tg);
  }
  return check_launch("warp3d_bwd_tile_kernel");
}

template <int TZ, int TY, int HALO, int METHOD, int CC = 1, bool ABS = false>
static int launch_tile(const float* vol, const float* flow, float* out, TileGeo tg, int H, int W, int src_n0,
                       int out_n0, cudaStream_t st) {
  using Cfg = TileCfg<TZ, TY, HALO, CC>;
  tg.ntz = (out_n0 + TZ - 1) / TZ; tg.nty = (H + TY - 1) / TY; tg.ntx = (W + Cfg::TX - 1) / Cfg::TX;
  if ((int64_t)tg.B * tg.ntz > 65535 || tg.nty > 65535 || Cfg::SMEM > 227 * 1024) return 1;   // caller falls back
  tg.g.C = CC;
  CUtensorMap tmv, tmf;
  const uint64_t vd[4] = {(uint64_t)W * CC, (uint64_t)H, (uint64_t)src_n0, (uint64_t)tg.B};
  const uint32_t vb[4] = {(uint32_t)(Cfg::BX * CC), (uint32_t)Cfg::BY, (uint32_t)Cfg::BZ, 1};
  const uint64_t fd[4] = {(uint64_t)W * 3, (uint64_t)H, (uint64_t)out_n0, (uint64_t)tg.B};
  const uint32_t fb[4] = {(uint32_t)Cfg::TX * 3, (uint32_t)TY, (uint32_t)TZ, 1};
  int rc = encode_f32_4d(&tmv, vol, vd, vb, (uint64_t)tg.src_batch_stride);
  if (rc != NRT_OK) return rc;
  rc = encode_f32_4d(&tmf, flow, fd, fb, (uint64_t)tg.flow_bstride);
  if (rc != NRT_OK) return rc;
  auto kern = warp3d_tile_kernel<TZ, TY, HALO, METHOD, CC, ABS>;
  // set on every launch: the attribute is per device and the call costs ~1 us of host time
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM) != cudaSuccess)
    return check_launch("cudaFuncSetAttribute(warp3d_tile)");
  const dim3 grid(tg.ntx, tg.nty, tg.ntz * tg.B);
  kern<<<grid, Cfg::NW * 32, Cfg::SMEM, st>>>(tmv, tmf, vol, out, tg, env_int("NRT_WARP_FOLLOW", 1));
  return check_launch("warp3d_tile_kernel");
}

template <int D, int METHOD>
static int launch_warp_generic(const float* vol, const float* flow, float* out, const WarpGeo& wg, cudaStream_t st) {
  const bool vec = (wg.g.C % 4 == 0) && aligned16(vol) && aligned16(out) && ((wg.src_batch_stride | wg.out_bstride) & 3) == 0;
  const int64_t total = (int64_t)wg.B * wg.out_vox * (vec ? wg.g.C / 4 : 1);
  if (total == 0) return NRT_OK;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 32);
  if (vec) warp_generic_kernel<D, 4, METHOD><<<grid, 256, 0, st>>>(vol, flow, out, wg);
  else warp_generic_kernel<D, 1, METHOD><<<grid, 256, 0, st>>>(vol, flow, out, wg);
  return check_launch("warp_generic_kernel");
}

template <int D, int METHOD>
static int launch_interpn(const float* vol, const Geo& g, const float* loc, int64_t n_out, float* out, cudaStream_t st) {
  const bool vec = (g.C % 4 == 0) && aligned16(vol) && aligned16(out);
  const int64_t total = n_out * (vec ? g.C / 4 : 1);
  if (total == 0) return NRT_OK;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 32);
  if (vec) interpn_kernel<D, 4, METHOD><<<grid, 256, 0, st>>>(vol, g, loc, n_out, out);
  else interpn_kernel<D, 1, METHOD><<<grid, 256, 0, st>>>(vol, g, loc, n_out, out);
  return check_launch("interpn_kernel");
}

template <int D, int METHOD>
static int launch_resize(const float* vol, float* out, const ResizeGeo& rg, cudaStream_t st) {
  const bool vec = (rg.g.C % 4 == 0) && aligned16(vol) && aligned16(out);
  const int64_t total = (int64_t)rg.B * rg.out_vox * (vec ? rg.g.C / 4 : 1);
  if (total == 0) return NRT_OK;
  const int grid = (int)imin64((total + 255) / 256, (int64_t)sm_count() * 32);
  if (vec) resize_kernel<D, 4, METHOD><<<grid, 256, 0, st>>>(vol, out, rg);
  else resize_kernel<D, 1, METHOD><<<grid, 256, 0, st>>>(vol, out, rg);
  return check_launch("resize_kernel");
}

#define NRT_DISPATCH_D_METHOD(D, method, CALL)                                  \
  do {                                                                          \
    if ((method) == NRT_LINEAR) {                                               \
      if ((D) == 1) return CALL(1, NRT_LINEAR);                                 \
      if ((D) == 2) return CALL(2, NRT_LINEAR);                                 \
      return CALL(3, NRT_LINEAR);                                               \
    } else {                                                                    \
      if ((D) == 1) return CALL(1, NRT_NEAREST);                                \
      if ((D) == 2) return CALL(2, NRT_NEAREST);                                \
      return CALL(3, NRT_NEAREST);                                              \
    }                                                                           \
  } while (0)

static int check_common(int D, int C, int method) {
  NRT_REQUIRE(D >= 1 && D <= 3, NRT_E_ARG, "D must be 1, 2 or 3 (got %d)", D);
  NRT_REQUIRE(C >= 1, NRT_E_ARG, "C must be >= 1 (got %d)", C);
  NRT_REQUIRE(method == NRT_LINEAR || method == NRT_NEAREST, NRT_E_ARG,
              "method should be linear or nearest, got: %d", method);
  return NRT_OK;
}

static int try_tile_path(const float* vol, const float* flow, float* out, int B, const int32_t* shape, int C,
                         int method, int has_fill, float fill, int src_z0, int src_n0, int out_z0,
                         int out_n0, int halo, int32_t* err_flag, cudaStream_t st, bool* used, int abs_loc = 0,
                         int64_t vbs = 0, int64_t fbs = 0, int64_t obs = 0) {
  *used = false;
  const int H = shape[1], W = shape[2];
  if (env_int("NRT_WARP_TILE", 1) == 0) return NRT_OK;
  if (W % 4 != 0 || !aligned16(vol) || !aligned16(flow) || !aligned16(out) || W < 32) return NRT_OK;
  // C = 1 runs 8x8x32 tiles (4 CTAs per SM); `halo` picks the smallest built halo that covers it
  if (halo <= 0) halo = 3;
  const int hsel = halo <= 3 ? 3 : (halo <= 4 ? 4 : (halo <= 6 ? 6 : 8));
  TileGeo tg;
  tg.g.S[0] = shape[0]; tg.g.S[1] = H; tg.g.S[2] = W;
  tg.g.src_z0 = src_z0; tg.g.src_n0 = src_n0; tg.g.C = 1;
  tg.g.has_fill = has_fill; tg.g.fill = fill; tg.g.err = err_flag;
  tg.out_z0 = out_z0; tg.out_n0 = out_n0; tg.B = B;
  tg.ntz = tg.nty = tg.ntx = 0;
  tg.abs_loc = abs_loc;
  tg.out_vox = (int64_t)out_n0 * H * W;
  tg.src_batch_stride = vbs ? vbs : (int64_t)src_n0 * H * W * C;
  tg.flow_bstride = fbs ? fbs : tg.out_vox * 3;
  tg.out_bstride = obs ? obs : tg.out_vox * C;
  if ((tg.src_batch_stride | tg.flow_bstride | tg.out_bstride) & 3) return NRT_OK;   // TMA strides: multiples of 16 bytes
  int rc = 1;
  if (abs_loc) {
    // absolute locations: instantiated for the default tile shapes only (other shapes: generic gather kernel)
#define NRT_TILE_ABS(cc, tz)                                                                                 \
    if (C == (cc))                                                                                           \
      rc = method == NRT_LINEAR                                                                              \
               ? launch_tile<tz, 8, 3, NRT_LINEAR, cc, true>(vol, flow, out, tg, H, W, src_n0, out_n0, st)   \
               : launch_tile<tz, 8, 3, NRT_NEAREST, cc, true>(vol, flow, out, tg, H, W, src_n0, out_n0, st);
    NRT_TILE_ABS(1, 8) NRT_TILE_ABS(2, 4) NRT_TILE_ABS(3, 4) NRT_TILE_ABS(4, 4)
#undef NRT_TILE_ABS
    if (rc == 1) return NRT_OK;
    *used = true;
    return rc;
  }
  if (C > 1) {
    // 2-4 channels: (x, channel) is one contiguous TMA dimension; 4x8x32 tiles keep the
    // staged box (22 KB per channel) small enough for two CTAs per SM
#define NRT_TILE_C(cc)                                                                                   \
    if (C == (cc))                                                                                       \
      rc = method == NRT_LINEAR                                                                          \
               ? launch_tile<4, 8, 3, NRT_LINEAR, cc>(vol, flow, out, tg, H, W, src_n0, out_n0, st)  \
               : launch_tile<4, 8, 3, NRT_NEAREST, cc>(vol, flow, out, tg, H, W, src_n0, out_n0, st);
    NRT_TILE_C(2) NRT_TILE_C(3) NRT_TILE_C(4)
#undef NRT_TILE_C
    if (rc == 1) return NRT_OK;
    *used = true;
    return rc;
  }
#define NRT_TILE_CASE(hh)                                                                                \
  if (hsel == (hh))                                                                                      \
    rc = method == NRT_LINEAR                                                                            \
             ? launch_tile<8, 8, hh, NRT_LINEAR>(vol, flow, out, tg, H, W, src_n0, out_n0, st)           \
             : launch_tile<8, 8, hh, NRT_NEAREST>(vol, flow, out, tg, H, W, src_n0, out_n0, st);
  NRT_TILE_CASE(3) NRT_TILE_CASE(4) NRT_TILE_CASE(6) NRT_TILE_CASE(8)
#undef NRT_TILE_CASE
  if (rc == 1) return NRT_OK;                              // not launched: fall back
  *used = true;
  return rc;
}

}  // namespace nrt

using namespace nrt;

extern "C" {

int nrt_interpn_f32(const float* vol, const int32_t* vol_shape, int D, int C, const float* loc,
                    int64_t n_out, int method, int has_fill, float fill, float* out, void* stream) {
  // the reference's interpn takes any number of dimensions (utils.py:106-120); the gather kernel is instantiated for
  // D = 1..5 (2^D corners per point), the warp / resize entry points for the D <= 3 of the layers that call them
  NRT_REQUIRE(D >= 1 && D <= 5, NRT_E_ARG, "D must be 1..5 (got %d)", D);
  int rc = check_common(D <= 3 ? D : 3, C, method);
  if (rc != NRT_OK) return rc;
  NRT_REQUIRE(vol && vol_shape && out && (loc || n_out == 0), NRT_E_ARG, "null pointer");
  NRT_REQUIRE(n_out >= 0, NRT_E_ARG, "n_out < 0");
  Geo g;
  int64_t nvox = 1;
  for (int d = 0; d < 5; ++d) {
    g.S[d] = d < D ? vol_shape[d] : 1;
    NRT_REQUIRE(g.S[d] >= 1, NRT_E_ARG, "vol_shape[%d] = %d", d, g.S[d]);
    nvox *= g.S[d];
  }
  NRT_REQUIRE(nvox <= 0x7fffffffLL, NRT_E_SIZE, "volume has %lld voxels (> int32)", (long long)nvox);
  g.src_z0 = 0; g.src_n0 = g.S[0]; g.C = C; g.has_fill = has_fill; g.fill = fill; g.err = nullptr;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (D == 4) return method == NRT_LINEAR ? launch_interpn<4, NRT_LINEAR>(vol, g, loc, n_out, out, st)
                                          : launch_interpn<4, NRT_NEAREST>(vol, g, loc, n_out, out, st);
  if (D == 5) return method == NRT_LINEAR ? launch_interpn<5, NRT_LINEAR>(vol, g, loc, n_out, out, st)
                                          : launch_interpn<5, NRT_NEAREST>(vol, g, loc, n_out, out, st);
#define CALL(DD, MM) launch_interpn<DD, MM>(vol, g, loc, n_out, out, st)
  NRT_DISPATCH_D_METHOD(D, method, CALL);
#undef CALL
}

int nrt_interpn_grid_f32(const float* vol, const float* loc, float* out, const int32_t* shape, int C, int method,
                         int has_fill, float fill, int halo, void* stream) {
  int rc = check_common(3, C, method);
  if (rc != NRT_OK) return rc;
  NRT_REQUIRE(vol && loc && out && shape, NRT_E_ARG, "null pointer");
  int64_t nvox = 1;
  for (int d = 0; d < 3; ++d) {
    NRT_REQUIRE(shape[d] >= 1, NRT_E_ARG, "shape[%d] = %d", d, shape[d]);
    nvox *= shape[d];
  }
  NRT_REQUIRE(nvox <= 0x7fffffffLL, NRT_E_SIZE, "volume has %lld voxels (> int32)", (long long)nvox);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (C <= 4) {
    bool used = false;
    rc = try_tile_path(vol, loc, out, 1, shape, C, method, has_fill, fill, 0, shape[0], 0, shape[0], halo, nullptr,
                       st, &used, /*abs_loc=*/1);
    if (rc != NRT_OK || used) return rc;
  }
  return nrt_interpn_f32(vol, shape, 3, C, loc, nvox, method, has_fill, fill, out, stream);
}

static int warp_impl(const float* vol, const float* flow, float* out, int B, const int32_t* shape, int D,
                     int C, int method, int has_fill, float fill, int src_z0, int src_n0, int out_z0,
                     int out_n0, int halo, int32_t* err_flag, int64_t vbs, int64_t fbs, int64_t obs, void* stream) {
  int rc = check_common(D, C, method);
  if (rc != NRT_OK) return rc;
  NRT_REQUIRE(vol && flow && out && shape, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 0, NRT_E_ARG, "B < 0");
  WarpGeo wg;
  int64_t plane = 1;
  for (int d = 0; d < 3; ++d) {
    wg.g.S[d] = d < D ? shape[d] : 1;
    NRT_REQUIRE(wg.g.S[d] >= 1, NRT_E_ARG, "shape[%d] = %d", d, wg.g.S[d]);
    if (d > 0) plane *= wg.g.S[d];
  }
  NRT_REQUIRE(src_z0 >= 0 && src_n0 >= 1 && src_z0 + src_n0 <= shape[0], NRT_E_ARG,
              "resident source planes [%d,%d) outside [0,%d)", src_z0, src_z0 + src_n0, shape[0]);
  NRT_REQUIRE(out_z0 >= 0 && out_n0 >= 0 && out_z0 + out_n0 <= shape[0], NRT_E_ARG,
              "output planes [%d,%d) outside [0,%d)", out_z0, out_z0 + out_n0, shape[0]);
  NRT_REQUIRE(plane * src_n0 <= 0x7fffffffLL && plane * out_n0 * 3 <= 0x7fffffffLL * 4, NRT_E_SIZE,
              "slab too large for int32 indexing");
  NRT_REQUIRE(vbs >= 0 && fbs >= 0 && obs >= 0, NRT_E_ARG, "negative batch stride");
  NRT_REQUIRE((vbs == 0 || vbs >= plane * src_n0 * C) && (fbs == 0 || fbs >= plane * out_n0 * D) &&
              (obs == 0 || obs >= plane * out_n0 * C), NRT_E_ARG, "batch stride smaller than one batch item");
  if (B == 0 || out_n0 == 0) return NRT_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // 3 or more channels: z-marching ring kernel (all channels of a voxel side by side in shared memory); C = 2 stays
  // on the box tiles, whose halo is still small at two channels.
  if (D == 3 && C >= 3) {
    bool used = false;
    rc = warp3d_march(vol, flow, out, B, shape, C, method, has_fill, fill, src_z0, src_n0, out_z0, out_n0,
                      halo, err_flag, vbs, fbs, obs, st, &used);
    if (rc != NRT_OK || used) return rc;
  }
  if (D == 3 && C <= 4) {
    bool used = false;
    rc = try_tile_path(vol, flow, out, B, shape, C, method, has_fill, fill, src_z0, src_n0, out_z0, out_n0,
                       halo, err_flag, st, &used, 0, vbs, fbs, obs);
    if (rc != NRT_OK || used) return rc;
  }
  wg.g.src_z0 = src_z0; wg.g.src_n0 = src_n0; wg.g.C = C;
  wg.g.has_fill = has_fill; wg.g.fill = fill; wg.g.err = err_flag;
  wg.out_z0 = out_z0; wg.out_n0 = out_n0; wg.B = B;
  wg.out_vox = plane * out_n0;
  wg.src_batch_stride = vbs ? vbs : plane * src_n0 * C;
  wg.flow_bstride = fbs ? fbs : wg.out_vox * D;
  wg.out_bstride = obs ? obs : wg.out_vox * C;
#define CALL(DD, MM) launch_warp_generic<DD, MM>(vol, flow, out, wg, st)
  NRT_DISPATCH_D_METHOD(D, method, CALL);
#undef CALL
}

int nrt_warp_f32(const float* vol, const float* flow, float* out, int B, const int32_t* shape, int D,
                 int C, int method, int has_fill, float fill, int src_z0, int src_n0, int out_z0,
                 int out_n0, int halo, int32_t* err_flag, void* stream) {
  return warp_impl(vol, flow, out, B, shape, D, C, method, has_fill, fill, src_z0, src_n0, out_z0, out_n0, halo,
                   err_flag, 0, 0, 0, stream);
}

int nrt_warp_strided_f32(const float* vol, const float* flow, float* out, int B, const int32_t* shape, int D,
                         int C, int method, int has_fill, float fill, int src_z0, int src_n0, int out_z0,
                         int out_n0, int halo, int32_t* err_flag, int64_t vol_batch_stride,
                         int64_t flow_batch_stride, int64_t out_batch_stride, void* stream) {
  return warp_impl(vol, flow, out, B, shape, D, C, method, has_fill, fill, src_z0, src_n0, out_z0, out_n0, halo,
                   err_flag, vol_batch_stride, flow_batch_stride, out_batch_stride, stream);
}

int nrt_resize_f32(const float* vol, float* out, int B, const int32_t* in_shape, const int32_t* out_shape,
                   int D, int C, int method, int out_z0, int out_n0, void* stream) {
  int rc = check_common(D, C, method);
  if (rc != NRT_OK) return rc;
  NRT_REQUIRE(vol && out && in_shape && out_shape, NRT_E_ARG, "null pointer");
  NRT_REQUIRE(B >= 0, NRT_E_ARG, "B < 0");
  ResizeGeo rg;
  int64_t in_vox = 1, out_plane = 1;
  for (int d = 0; d < 3; ++d) {
    rg.g.S[d] = d < D ? in_shape[d] : 1;
    rg.M[d] = d < D ? out_shape[d] : 1;
    NRT_REQUIRE(rg.g.S[d] >= 1 && rg.M[d] >= 0, NRT_E_ARG, "bad shape at axis %d", d);
    // tf.linspace in fp32: delta = (stop - start) / (num - 1)
    rg.delta[d] = rg.M[d] > 1 ? (float)(rg.g.S[d] - 1) / (float)(rg.M[d] - 1) : 0.0f;
    in_vox *= rg.g.S[d];
    if (d > 0) out_plane *= rg.M[d];
  }
  NRT_REQUIRE(out_z0 >= 0 && out_n0 >= 0 && out_z0 + out_n0 <= rg.M[0], NRT_E_ARG, "output planes out of range");
  NRT_REQUIRE(in_vox <= 0x7fffffffLL && out_plane * out_n0 <= 0x7fffffffLL, NRT_E_SIZE, "volume too large for int32 indexing");
  rg.g.src_z0 = 0; rg.g.src_n0 = rg.g.S[0]; rg.g.C = C; rg.g.has_fill = 0; rg.g.fill = 0.f; rg.g.err = nullptr;
  rg.out_z0 = out_z0; rg.out_n0 = out_n0; rg.B = B;
  rg.src_batch_stride = in_vox * C;
  rg.out_vox = out_plane * out_n0;
  if (B == 0 || rg.out_vox == 0) return NRT_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (D == 3 && in_vox * C <= 0x7fffffffLL && env_int("NRT_RESIZE_GENERIC", 0) == 0) {
    // planes per CTA: 32 (fewer prologues and box waits per output plane); short slabs take fewer so that the grid
    // keeps a few waves
    int TZ = out_n0 >= 64 ? 32 : (out_n0 >= 24 ? 16 : 8);
    if (method != NRT_LINEAR || C < 1 || C > 4) TZ = 8;          // the marching path is linear, C = 1..4
    // up-sampling: source box of every output tile staged by TMA (resize3d_tile_kernel)
    if (method == NRT_LINEAR && C >= 1 && C <= 4 && env_int("NRT_RESIZE_TILE", 1) && aligned16(vol) &&
        (rg.g.S[2] * C) % 4 == 0 && ((C != 2 && C != 4) || (reinterpret_cast<uintptr_t>(out) & (C == 4 ? 15u : 7u)) == 0)) {
      const int xalign = (C == 4) ? 1 : (C == 2 ? 2 : 4);
      // voxel-pair kernel (16-row tiles; NRT_RESIZE_TILE_X2=0: one voxel per thread): needs an even row pitch / aligned
      // output for its 64 / 128-bit stores.  It runs 2 CTAs per SM (registers) and can afford a 100 KB box.
      const bool x2 = env_int("NRT_RESIZE_TILE_X2", 1) != 0 && (rg.M[2] * C) % (C == 2 ? 4 : 2) == 0 &&
                      (reinterpret_cast<uintptr_t>(out) & 15u) == 0 && (rg.out_vox * C) % 4 == 0;
      const size_t box_budget = (x2 ? 100 : 72) * 1024;
      const int unstaged = env_int("NRT_RESIZE_UNSTAGED", 0);      // test hook: every CTA takes its global-memory path
      const int tyt = x2 ? 16 : 8;
      ResizeBox bxs;
      bxs.by = resize_axis_extent(rg.g.S[1], rg.M[1], rg.delta[1], 0, rg.M[1], tyt, 1);
      bxs.bx = resize_axis_extent(rg.g.S[2], rg.M[2], rg.delta[2], 0, rg.M[2], 32, xalign);
      bxs.bx = (bxs.bx + xalign - 1) / xalign * xalign;
      bxs.bz = resize_axis_extent(rg.g.S[0], rg.M[0], rg.delta[0], out_z0, out_n0, TZ, 1);
      const size_t box_bytes = (size_t)bxs.bz * bxs.by * bxs.bx * C * 4;
      const int ntz3 = (out_n0 + TZ - 1) / TZ, nty3 = (rg.M[1] + tyt - 1) / tyt, ntx3 = (rg.M[2] + 31) / 32;
      const int64_t grid3 = (int64_t)B * ntz3 * nty3 * ntx3;
      if (box_bytes <= box_budget && bxs.bx * C <= 256 && bxs.by <= 256 && bxs.bz <= 256 && grid3 <= 0x7fffffffLL) {
        CUtensorMap tmv;
        const uint64_t vd[4] = {(uint64_t)rg.g.S[2] * C, (uint64_t)rg.g.S[1], (uint64_t)rg.g.S[0], (uint64_t)B};
        const uint32_t vb[4] = {(uint32_t)(bxs.bx * C), (uint32_t)bxs.by, (uint32_t)bxs.bz, 1};
        int erc = encode_f32_4d(&tmv, vol, vd, vb);
        if (erc != NRT_OK) return erc;
        const size_t smem = ((box_bytes + 15) & ~(size_t)15) + 32;
        const float nzf = -0.0f, onef = 1.0f;
        uint32_t nzb, oneb;
        memcpy(&nzb, &nzf, 4); memcpy(&oneb, &onef, 4);
        const f32x2 negzero2 = ((f32x2)nzb << 32) | nzb, one2 = ((f32x2)oneb << 32) | oneb;
#define NRT_RESIZE_TILE(CT, TZZ)                                                                                          \
        do {                                                                                                              \
          if (x2) {                                                                                                       \
            auto kern = resize3d_pair_kernel<CT, TZZ>;                                                                    \
            if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)        \
              return check_launch("cudaFuncSetAttribute(resize3d_pair)");                                                 \
            kern<<<(int)grid3, 256, smem, st>>>(tmv, vol, out, rg, bxs, ntz3, nty3, ntx3, xalign, negzero2, one2,         \
                                                unstaged);                                                                \
          } else {                                                                                                        \
            auto kern = resize3d_tile_kernel<CT, TZZ>;                                                                    \
            if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)        \
              return check_launch("cudaFuncSetAttribute(resize3d_tile)");                                                 \
            kern<<<(int)grid3, 256, smem, st>>>(tmv, vol, out, rg, bxs, ntz3, nty3, ntx3, xalign);                        \
          }                                                                                                               \
        } while (0)
#define NRT_RESIZE_TILE_C(CT)                                                                                             \
        do { if (TZ == 8) NRT_RESIZE_TILE(CT, 8); else if (TZ == 16) NRT_RESIZE_TILE(CT, 16); else NRT_RESIZE_TILE(CT, 32); } while (0)
        switch (C) {
          case 1: NRT_RESIZE_TILE_C(1); break;
          case 2: NRT_RESIZE_TILE_C(2); break;
          case 3: NRT_RESIZE_TILE_C(3); break;
          default: NRT_RESIZE_TILE_C(4); break;
        }
#undef NRT_RESIZE_TILE_C
#undef NRT_RESIZE_TILE
        return check_launch("resize3d_tile_kernel");
      }
    }
    const int ntz = (out_n0 + TZ - 1) / TZ, nty = (rg.M[1] + 7) / 8, ntx = (rg.M[2] + 31) / 32;
    const int64_t grid = (int64_t)B * ntz * nty * ntx;
    if (grid <= 0x7fffffffLL) {
#define NRT_RESIZE3D(CT)                                                                              \
      do {                                                                                            \
        if (method != NRT_LINEAR) resize3d_kernel<NRT_NEAREST, CT><<<(int)grid, 256, 0, st>>>(vol, out, rg, ntz, nty, ntx);  \
        else if (TZ == 16) resize3d_kernel<NRT_LINEAR, CT, 16><<<(int)grid, 256, 0, st>>>(vol, out, rg, ntz, nty, ntx);     \
        else if (TZ == 32) resize3d_kernel<NRT_LINEAR, CT, 32><<<(int)grid, 256, 0, st>>>(vol, out, rg, ntz, nty, ntx);     \
        else resize3d_kernel<NRT_LINEAR, CT><<<(int)grid, 256, 0, st>>>(vol, out, rg, ntz, nty, ntx); \
      } while (0)
      // the C = 2 / 4 kernels store float2 / float4 per voxel: fall back to the run-time-C kernel for an unaligned output
      const bool al = (reinterpret_cast<uintptr_t>(out) & (C == 4 ? 15u : 7u)) == 0;
      switch ((C == 2 || C == 4) && !al ? 0 : C) {
        case 1: NRT_RESIZE3D(1); break;
        case 2: NRT_RESIZE3D(2); break;
        case 3: NRT_RESIZE3D(3); break;
        case 4: NRT_RESIZE3D(4); break;
        default: NRT_RESIZE3D(0); break;
      }
#undef NRT_RESIZE3D
      return check_launch("resize3d_kernel");
    }
  }
#define CALL(DD, MM) launch_resize<DD, MM>(vol, out, rg, st)
  NRT_DISPATCH_D_METHOD(D, method, CALL);
#undef CALL
}

}  // extern "C"
