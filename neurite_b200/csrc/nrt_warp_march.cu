// nrt_warp_march.cu -- dense warp (identity grid + flow -> interpn, reference utils.py:73-220 under the voxelmorph
// SpatialTransformer contract) for MULTI-CHANNEL volumes, D = 3.  This is the 16-label softmax warp of
// BASELINE.json configs[4] (call sites neurite/tf/models.py:806-807, 1157-1159).
//
// Why a second kernel: the box-tile kernel (nrt_interp.cu) stages tile + halo in all three axes.  With C channels a
// voxel is 4C bytes, the tile that fits shared memory shrinks and the halo dominates: a 4x8x32 tile with halo 3 reads
// 5.5 box voxels per output voxel, and a 16-channel box does not fit at all.  Here a CTA owns a (y, x) COLUMN of the
// output and MARCHES along z with a ring of source planes in shared memory: every source plane of the column is
// loaded once (TMA, one mbarrier per ring slot), so the halo is paid in y and x only (2.4 staged voxels per output
// voxel for 16 channels) and all channels of a voxel sit side by side, i.e. a corner is ONE 16-byte shared-memory
// load per lane and four lanes cover a 16-channel voxel.
//
//   ring slot  = [BY][BX][CCH] source plane box  +  [TY][TX][3] flow tile of the output plane that becomes
//                computable when this source plane lands (the last plane of its window)
//   producer   = one thread of an extra warp: waits for a slot's `empty` barrier, arms `full`, issues the two TMA loads
//   consumers  = NW warps; item = (voxel of the plane tile, 4-channel quad); per output plane a warp waits only for
//                the newest plane of the window, computes, and releases the oldest plane -- no block-wide barrier
//
// Arithmetic is the reference's (separately rounded multiplies / adds, itertools.product corner order); a voxel
// whose corners are not all inside the staged window falls back to the global gather (same code as the generic
// kernel), so results never depend on tile, halo or ring geometry.
#include "nrt_interp.cuh"

namespace nrt {

struct MarchGeo {
  Geo g;                        // S = full extents, src_z0 / src_n0 = resident source planes, C = TOTAL channels
  int out_z0, out_n0;           // produced planes of axis 0 (global start, count)
  int B, nchunk, nseg, seg_len; // channel chunks of CCH, z segments per column and their length
  int64_t src_batch_stride, out_vox;
  int64_t flow_bstride, out_bstride;   // elements between batch items of flow / out
};

// CCH = channels staged per voxel (a chunk of the volume's C); VEC: lanes own 4-channel quads, else all CCH channels.
// QPT = quads per thread (VEC only): the per-voxel corner setup (~60 instructions) and the 8 corner weights are
// shared by the QPT quads a thread owns -- with one quad per thread they are 2/3 of all instructions.
// The ring holds the window of one output plane plus AHEAD planes of prefetch.
template <int CCH, int TY_, int TX_, int HALO_, int AHEAD_, int QPT_ = 1>
struct MarchCfg {
  static constexpr int TY = TY_, TX = TX_, HALO = HALO_, AHEAD = AHEAD_;
  static constexpr bool VEC = (CCH % 4 == 0);
  static constexpr int QPT = VEC ? QPT_ : 1;
  static constexpr int Q = VEC ? CCH / 4 : 1;                   // quads per voxel
  static constexpr int LPV = VEC ? Q / QPT : 1;                 // lanes per voxel
  static constexpr int CPL = VEC ? 4 : CCH;                     // channels per lane and pass
  static_assert(!VEC || Q % QPT == 0, "quads per thread must divide the quads per voxel");
  // the TMA needs a 16-byte aligned start address: (x0 - HX) * C * 4 bytes
  static constexpr int HX = VEC ? HALO : ((HALO + 3) & ~3);
  static constexpr int BY = TY + 2 * HALO, BX = TX + 2 * HX;
  static constexpr int WIN = 2 * HALO + 1;                      // source planes one output plane can touch
  static constexpr int R = WIN + AHEAD;                         // ring slots
  static constexpr int BOX_ELEMS = BY * BX * CCH, FLOW_ELEMS = TY * TX * 3;
  static constexpr int BOX_BYTES = BOX_ELEMS * 4, FLOW_BYTES = FLOW_ELEMS * 4;
  static constexpr int FLOW_OFF = (BOX_BYTES + 127) & ~127;     // byte offset of the flow tile inside a slot
  static constexpr int SLOT_BYTES = (FLOW_OFF + FLOW_BYTES + 127) & ~127;
  static constexpr size_t SMEM = (size_t)R * SLOT_BYTES + 2 * R * sizeof(uint64_t);
  static constexpr int ITEMS = TY * TX * LPV;
  static_assert(BX <= 256 && BY <= 256 && (VEC || BX * CCH <= 256), "TMA box limit");
  static_assert((BX * CCH) % 4 == 0 && (TX * 3) % 4 == 0, "TMA inner box must be a multiple of 16 bytes");
};

template <int CPL>
__device__ __forceinline__ void lds_channels(const float* p, float (&v)[CPL]) {
  if (CPL == 4) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    v[0] = q.x; v[1 % CPL] = q.y; v[2 % CPL] = q.z; v[3 % CPL] = q.w;
  } else {
#pragma unroll
    for (int c = 0; c < CPL; ++c) v[c] = p[c];
  }
}

template <int CCH, int TY, int TX, int HALO, int AHEAD, int NW, int METHOD, int QPT = 1>
__global__ void __launch_bounds__((NW + 1) * 32, 1)
warp3d_march_kernel(const __grid_constant__ CUtensorMap tm_vol, const __grid_constant__ CUtensorMap tm_flow,
                    const float* __restrict__ vol, float* __restrict__ out, MarchGeo w) {
  using Cfg = MarchCfg<CCH, TY, TX, HALO, AHEAD, QPT>;
  constexpr int R = Cfg::R, WIN = Cfg::WIN, BX = Cfg::BX, BY = Cfg::BY, LPV = Cfg::LPV, CPL = Cfg::CPL, Q = Cfg::Q;
  constexpr int NTC = NW * 32;
  static_assert(Cfg::ITEMS % NTC == 0, "the plane tile must be a whole number of passes of the consumer threads");
  constexpr int ITER = Cfg::ITEMS / NTC;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)R * Cfg::SLOT_BYTES);
  uint64_t* empty = full + R;
  const Geo& g = w.g;
  const int H = g.S[1], W = g.S[2], Ctot = g.C;
  const int tid = threadIdx.x, wid = tid >> 5, lane = tid & 31;
  const int x0 = blockIdx.x * TX, y0 = blockIdx.y * TY;
  int zb = blockIdx.z;
  const int seg = zb % w.nseg; zb /= w.nseg;
  const int chunk = zb % w.nchunk;
  const int b = zb / w.nchunk;
  const int zs = seg * w.seg_len;                               // first produced plane of this CTA (slab-local)
  const int nz = min(w.seg_len, w.out_n0 - zs);
  const int p_first = w.out_z0 + zs - HALO;                     // global source plane of ring index 0
  const int n_planes = nz + 2 * HALO;
  if (tid == 0) {
    for (int s = 0; s < R; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, NW); }
    fence_mbar_init();
  }
  __syncthreads();

  if (wid == NW) {
    // ===== producer: ring index i carries source plane p_first + i and the flow tile of output plane zs + i - 2 HALO
    // (planes / tiles outside the tensors are zero-filled by the TMA and never read)
    if (lane == 0) {
      for (int i = 0; i < n_planes; ++i) {
        const int slot = i % R, round = i / R;
        if (round >= 1) mbar_wait(empty + slot, (uint32_t)((round - 1) & 1));
        unsigned char* dst = smem_raw + (size_t)slot * Cfg::SLOT_BYTES;
        mbar_expect_tx(full + slot, (uint32_t)(Cfg::BOX_BYTES + Cfg::FLOW_BYTES));
        const int pz = p_first + i - g.src_z0;
        if (Cfg::VEC) tma_load_5d(dst, &tm_vol, full + slot, chunk * CCH, x0 - Cfg::HX, y0 - HALO, pz, b);
        else tma_load_4d(dst, &tm_vol, full + slot, (x0 - Cfg::HX) * CCH, y0 - HALO, pz, b);
        tma_load_4d(dst + Cfg::FLOW_OFF, &tm_flow, full + slot, x0 * 3, y0, zs + i - 2 * HALO, b);
      }
    }
    return;
  }

  // ===== consumers =====
  const float* volb = vol + (size_t)b * w.src_batch_stride;
  float* outb = out + (size_t)b * w.out_bstride;
  const int c_base = chunk * CCH;
  const int oy = y0 - HALO, ox = x0 - Cfg::HX;
  const int lo_y = max(oy, 0), hi_y = min(oy + BY - 1, H - 1);
  const int lo_x = max(ox, 0), hi_x = min(ox + BX - 1, W - 1);
  const int res_lo = g.src_z0, res_hi = g.src_z0 + g.src_n0 - 1;
  // per-thread constants of its ITER items
  int vxs[ITER], vys[ITER], qs[ITER];
#pragma unroll
  for (int it = 0; it < ITER; ++it) {
    const int item = it * NTC + (tid % NTC);
    qs[it] = item % LPV;
    const int v = item / LPV;
    vxs[it] = v % TX; vys[it] = v / TX;
  }
  // every warp waits for every ring index in increasing order, so a barrier is never more than one phase ahead:
  // the first 2 HALO planes once, then the newest plane of each output plane's window
  for (int i = 0; i < 2 * HALO; ++i) mbar_wait(full + i, 0);
  for (int j = 0; j < nz; ++j) {
    const int inew = j + 2 * HALO;
    mbar_wait(full + (inew % R), (uint32_t)((inew / R) & 1));
    const int wbase = j % R;                                    // ring slot of the window's first plane
    const float* s_flow = reinterpret_cast<const float*>(smem_raw + (size_t)(inew % R) * Cfg::SLOT_BYTES + Cfg::FLOW_OFF);
    const int zl = zs + j, gz = w.out_z0 + zl;
    const int oz = gz - HALO;
    const int lo_z = max(oz, res_lo), hi_z = min(oz + WIN - 1, res_hi);
    const float fz = (float)gz;
#pragma unroll
    for (int it = 0; it < ITER; ++it) {
      const int vx = vxs[it], vy = vys[it], q = qs[it];
      const int gx = x0 + vx, gy = y0 + vy;
      const float* fl = s_flow + (vy * TX + vx) * 3;
      const float lz = __fadd_rn(fz, fl[0]);
      const float ly = __fadd_rn((float)gy, fl[1]);
      const float lx = __fadd_rn((float)gx, fl[2]);
      // Quads of this thread: q, q + LPV, q + 2 LPV, ... (interleaved: in one pass the LPV lanes of a voxel read LPV
      // ADJACENT quads, one contiguous 16 LPV-byte piece, so a quarter warp touches 8 / LPV pieces instead of 8
      // scattered quads -- fewer bank-group collisions for incoherent flows), visited in a rotated order so that
      // consecutive voxels -- a smooth flow -- hit distinct bank groups: a voxel is Q quads wide, 8 / Q voxels share a
      // 128-byte bank cycle, so voxel v starts at rotation v * Q / 8.
      const int rot = (Cfg::VEC && QPT > 1) ? (((vy * TX + vx) * Q) >> 3) : 0;
      float res[Cfg::QPT][CPL];
      bool ok;
      if (METHOD == NRT_LINEAR) {
        AxisBox<true, WIN> az; AxisBox<true, BY> ay; AxisBox<true, BX> ax;
        az.setup(lz, oz, lo_z, hi_z, g.S[0] - 1);
        ay.setup(ly, oy, lo_y, hi_y, H - 1);
        ax.setup(lx, ox, lo_x, hi_x, W - 1);
        ok = az.ok & ay.ok & ax.ok;
        int s0 = wbase + az.c0; s0 -= (s0 >= R) ? R : 0;
        int s1 = s0 + az.d;     s1 -= (s1 >= R) ? R : 0;
        const int inplane = (ay.c0 * BX + ax.c0) * CCH + q * CPL;
        const float* p0 = reinterpret_cast<const float*>(smem_raw + (size_t)s0 * Cfg::SLOT_BYTES) + inplane;
        const float* p1 = reinterpret_cast<const float*>(smem_raw + (size_t)s1 * Cfg::SLOT_BYTES) + inplane;
        const int dy = ay.d * BX * CCH, dx = ax.d * CCH;
        float k[8];
        corner_weights(az.wlo, az.whi, ay.wlo, ay.whi, ax.wlo, ax.whi, k);
#pragma unroll
        for (int qi = 0; qi < Cfg::QPT; ++qi) {
          const int qo = (Cfg::QPT > 1 ? ((qi + rot) % Cfg::QPT) : 0) * LPV * CPL;  // offset of this pass's quad
          float v[8][CPL];
          lds_channels<CPL>(p0 + qo, v[0]);           lds_channels<CPL>(p0 + qo + dx, v[1]);
          lds_channels<CPL>(p0 + qo + dy, v[2]);      lds_channels<CPL>(p0 + qo + dy + dx, v[3]);
          lds_channels<CPL>(p1 + qo, v[4]);           lds_channels<CPL>(p1 + qo + dx, v[5]);
          lds_channels<CPL>(p1 + qo + dy, v[6]);      lds_channels<CPL>(p1 + qo + dy + dx, v[7]);
#pragma unroll
          for (int c = 0; c < CPL; ++c) {
            float r = __fadd_rn(0.f, __fmul_rn(k[0], v[0][c]));
#pragma unroll
            for (int n = 1; n < 8; ++n) r = __fadd_rn(r, __fmul_rn(k[n], v[n][c]));
            res[qi][c] = r;
          }
        }
      } else {
        ok = true;
        const int cz = nearest_box<true, WIN>(lz, oz, lo_z, hi_z, g.S[0] - 1, ok);
        const int cy = nearest_box<true, BY>(ly, oy, lo_y, hi_y, H - 1, ok);
        const int cx = nearest_box<true, BX>(lx, ox, lo_x, hi_x, W - 1, ok);
        int s0 = wbase + cz; s0 -= (s0 >= R) ? R : 0;
        const float* p0 = reinterpret_cast<const float*>(smem_raw + (size_t)s0 * Cfg::SLOT_BYTES) +
                          (cy * BX + cx) * CCH + q * CPL;
#pragma unroll
        for (int qi = 0; qi < Cfg::QPT; ++qi)
          lds_channels<CPL>(p0 + (Cfg::QPT > 1 ? ((qi + rot) % Cfg::QPT) : 0) * LPV * CPL, res[qi]);
      }
      if (gx >= W || gy >= H) continue;                         // lanes of a partial tile (after the loads: no divergence above)
      float* op = outb + (((size_t)zl * H + gy) * W + gx) * Ctot + c_base + q * CPL;
      if (!ok) {
        // rare: a corner outside the staged window -> the generic global gather (identical semantics, incl. the
        // fill rule and the resident-plane check that raises the device error flag)
        const float loc[3] = {lz, ly, lx};
        Corners<3, METHOD> kc;
        setup_point<3, METHOD>(g, loc, kc);
        const bool oob = g.has_fill ? out_of_bounds<3>(g, loc) : false;
        if (CPL == 4) {
#pragma unroll
          for (int qi = 0; qi < Cfg::QPT; ++qi) {
            float r4[4];
            gather_point<3, 4, METHOD>(volb, g, kc, oob, c_base + (q + LPV * qi) * 4, r4);
            *reinterpret_cast<float4*>(op + LPV * qi * 4) = make_float4(r4[0], r4[1], r4[2], r4[3]);
          }
        } else {
#pragma unroll
          for (int c = 0; c < CPL; ++c) {
            float r1[1];
            gather_point<3, 1, METHOD>(volb, g, kc, oob, c_base + c, r1);
            op[c] = r1[0];
          }
        }
        continue;
      }
      if (g.has_fill) {
#pragma unroll
        for (int qi = 0; qi < Cfg::QPT; ++qi)
#pragma unroll
          for (int c = 0; c < CPL; ++c) res[qi][c] = fill_if_oob(g, res[qi][c], lz, ly, lx);
      }
      if (CPL == 4) {
#pragma unroll
        for (int qi = 0; qi < Cfg::QPT; ++qi) {
          const int qo = (Cfg::QPT > 1 ? ((qi + rot) % Cfg::QPT) : 0) * LPV * 4;
          *reinterpret_cast<float4*>(op + qo) = make_float4(res[qi][0], res[qi][1 % CPL], res[qi][2 % CPL], res[qi][3 % CPL]);
        }
      } else {
#pragma unroll
        for (int c = 0; c < CPL; ++c) op[c] = res[0][c];
      }
    }
    // this warp is done with the oldest plane of the window (its next output plane is j + 1)
    __syncwarp();
    if (lane == 0) mbar_arrive(empty + (j % R));
  }
}

template <int CCH, int TY, int TX, int HALO, int AHEAD, int NW, int METHOD, int QPT = 1>
static int launch_march(const float* vol, const float* flow, float* out, MarchGeo mg, cudaStream_t st) {
  using Cfg = MarchCfg<CCH, TY, TX, HALO, AHEAD, QPT>;
  static_assert(Cfg::SMEM <= 227 * 1024, "ring does not fit shared memory");
  const int H = mg.g.S[1], W = mg.g.S[2], C = mg.g.C;
  const int ntx = (W + TX - 1) / TX, nty = (H + TY - 1) / TY;
  mg.nchunk = C / CCH;
  // z segments: enough CTAs for ~4 waves of the SMs, but segments of >= 16 planes (each pays 2 HALO extra planes)
  const int64_t cols = (int64_t)ntx * nty * mg.B * mg.nchunk;
  int nseg = (int)imin64((4 * (int64_t)sm_count() + cols - 1) / cols, mg.out_n0 / 16 > 0 ? mg.out_n0 / 16 : 1);
  const int forced = env_int("NRT_MARCH_NSEG", 0);
  if (forced > 0) nseg = forced < mg.out_n0 ? forced : mg.out_n0;
  if (nseg < 1) nseg = 1;
  mg.seg_len = (mg.out_n0 + nseg - 1) / nseg;
  mg.nseg = (mg.out_n0 + mg.seg_len - 1) / mg.seg_len;
  const int64_t gz = (int64_t)mg.nseg * mg.nchunk * mg.B;
  if (gz > 65535 || nty > 65535) return 1;                       // caller falls back
  CUtensorMap tmv, tmf;
  int rc;
  if (Cfg::VEC) {
    const uint64_t vd[5] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)mg.g.src_n0, (uint64_t)mg.B};
    const uint32_t vb[5] = {(uint32_t)CCH, (uint32_t)Cfg::BX, (uint32_t)Cfg::BY, 1, 1};
    rc = encode_f32_tiled(&tmv, vol, 5, vd, vb, (uint64_t)mg.src_batch_stride);
  } else {
    const uint64_t vd[4] = {(uint64_t)W * C, (uint64_t)H, (uint64_t)mg.g.src_n0, (uint64_t)mg.B};
    const uint32_t vb[4] = {(uint32_t)(Cfg::BX * CCH), (uint32_t)Cfg::BY, 1, 1};
    rc = encode_f32_tiled(&tmv, vol, 4, vd, vb, (uint64_t)mg.src_batch_stride);
  }
  if (rc != NRT_OK) return rc;
  const uint64_t fd[4] = {(uint64_t)W * 3, (uint64_t)H, (uint64_t)mg.out_n0, (uint64_t)mg.B};
  const uint32_t fb[4] = {(uint32_t)TX * 3, (uint32_t)TY, 1, 1};
  rc = encode_f32_tiled(&tmf, flow, 4, fd, fb, (uint64_t)mg.flow_bstride);
  if (rc != NRT_OK) return rc;
  auto kern = warp3d_march_kernel<CCH, TY, TX, HALO, AHEAD, NW, METHOD, QPT>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM) != cudaSuccess)
    return check_launch("cudaFuncSetAttribute(warp3d_march)");
  const dim3 grid(ntx, nty, (unsigned)gz);
  kern<<<grid, (NW + 1) * 32, Cfg::SMEM, st>>>(tmv, tmf, vol, out, mg);
  return check_launch("warp3d_march_kernel");
}

// Multi-channel D = 3 warp through the z-marching ring kernel.  *used = false (and NRT_OK) when the shape is not
// covered: the caller then takes the box-tile or the generic gather path.
int warp3d_march(const float* vol, const float* flow, float* out, int B, const int32_t* shape, int C, int method,
                 int has_fill, float fill, int src_z0, int src_n0, int out_z0, int out_n0, int halo,
                 int32_t* err_flag, int64_t vbs, int64_t fbs, int64_t obs, cudaStream_t st, bool* used) {
  *used = false;
  const int H = shape[1], W = shape[2];
  if (env_int("NRT_WARP_MARCH", 1) == 0) return NRT_OK;
  if (halo > 3) return NRT_OK;                                   // built for halo 3 (the gather fallback keeps any flow correct)
  if (W % 4 != 0 || W < 16 || !aligned16(vol) || !aligned16(flow) || !aligned16(out)) return NRT_OK;
  MarchGeo mg;
  mg.g.S[0] = shape[0]; mg.g.S[1] = H; mg.g.S[2] = W;
  mg.g.src_z0 = src_z0; mg.g.src_n0 = src_n0; mg.g.C = C;
  mg.g.has_fill = has_fill; mg.g.fill = fill; mg.g.err = err_flag;
  mg.out_z0 = out_z0; mg.out_n0 = out_n0; mg.B = B;
  mg.nchunk = mg.nseg = mg.seg_len = 1;
  mg.out_vox = (int64_t)out_n0 * H * W;
  mg.src_batch_stride = vbs ? vbs : (int64_t)src_n0 * H * W * C;
  mg.flow_bstride = fbs ? fbs : mg.out_vox * 3;
  mg.out_bstride = obs ? obs : mg.out_vox * C;
  if ((mg.src_batch_stride | mg.flow_bstride | mg.out_bstride) & 3) return NRT_OK;   // TMA strides: multiples of 16 bytes
  const bool lin = method == NRT_LINEAR;
  int rc = 1;
  // 8 / 16-channel chunks: two quads per thread share the corner setup (i.i.d. flows are bank-conflict bound either way)
  if (C % 16 == 0)
    rc = lin ? launch_march<16, 8, 16, 3, 3, 8, NRT_LINEAR, 2>(vol, flow, out, mg, st)
             : launch_march<16, 8, 16, 3, 3, 8, NRT_NEAREST, 2>(vol, flow, out, mg, st);
  else if (C % 8 == 0)
    rc = lin ? launch_march<8, 8, 32, 3, 3, 8, NRT_LINEAR, 2>(vol, flow, out, mg, st)
             : launch_march<8, 8, 32, 3, 3, 8, NRT_NEAREST, 2>(vol, flow, out, mg, st);
  else if (C % 4 == 0)
    rc = lin ? launch_march<4, 16, 32, 3, 3, 16, NRT_LINEAR>(vol, flow, out, mg, st)
             : launch_march<4, 16, 32, 3, 3, 16, NRT_NEAREST>(vol, flow, out, mg, st);
  else if (C == 3)
    rc = lin ? launch_march<3, 8, 32, 3, 3, 8, NRT_LINEAR>(vol, flow, out, mg, st)
             : launch_march<3, 8, 32, 3, 3, 8, NRT_NEAREST>(vol, flow, out, mg, st);
  if (rc == 1) return NRT_OK;
  *used = true;
  return rc;
}

}  // namespace nrt
