/*
 * neurite_b200.h -- C ABI of libneurite_b200.so (hand-written CUDA for sm_90a).
 *
 * The reference (adalca/neurite @ 7c4b05e) has no FFI: its extension boundary is python
 * callables / Keras layers over TensorFlow ops (SURVEY.md 8b).  Each entry point below
 * replaces the TensorFlow op sequence of the cited reference function; the python package
 * neurite_b200 binds them with ctypes and re-exposes the reference signatures
 * (see INTEGRATION.md for the binding a maintainer would add on the reference side).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross the ABI.
 *   - every device pointer is caller-owned, contiguous, channels-last ([batch,*spatial,C]),
 *     fp32 (int32 where stated); inputs are const; no entry point allocates or frees
 *     device memory, and none synchronises the device.
 *   - `stream` is a cudaStream_t (CUstream) passed as void*; work is enqueued on it.
 *   - return value: NRT_OK or a negative nrt_status; nrt_last_error_string() gives the
 *     thread-local detail.  Nothing throws across the ABI.
 *   - index arithmetic follows the reference: row-major flat index (utils.py:1068-1082).
 *     Outputs with more than 2^31-1 elements per batch item are rejected (NRT_E_SIZE).
 */
#ifndef NEURITE_B200_H_
#define NEURITE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NRT_ABI_VERSION 2

#if defined(__GNUC__)
#define NRT_API __attribute__((visibility("default")))
#else
#define NRT_API
#endif

typedef enum {
  NRT_OK = 0,
  NRT_E_ARG = -1,     /* bad argument (null pointer, rank, method, shape)              */
  NRT_E_SIZE = -2,    /* size outside what the kernels index (int32 per batch item)    */
  NRT_E_LAUNCH = -3,  /* CUDA launch / runtime error (string has cudaGetErrorString)   */
  NRT_E_ALIGN = -4,   /* pointer not aligned as the entry point requires               */
  NRT_E_NODEV = -5    /* no usable sm_90 device / driver                               */
} nrt_status;

enum { NRT_LINEAR = 0, NRT_NEAREST = 1 };
enum { NRT_ACT_LINEAR = 0, NRT_ACT_RELU = 1, NRT_ACT_SIGMOID = 2, NRT_ACT_TANH = 3 };
enum { NRT_STAT_SD = 0, NRT_STAT_MAX = 1, NRT_STAT_ABSMAX = 2, NRT_STAT_MINMAX = 3 };

NRT_API int nrt_version(void);
NRT_API const char* nrt_last_error_string(void);
NRT_API const char* nrt_status_string(int status);

/* ---------------------------------------------------------------------------------------
 * interpn -- replaces neurite/tf/utils/utils.py:73-220 (interpn).
 *   vol  [S_0..S_{D-1}, C]   loc [n_out, D]   out [n_out, C]      D in 1..5
 *   method NRT_LINEAR: clip / floor / 2^D-corner gather in itertools.product order with
 *   weights ((w0*w1)*w2), separate mul and add roundings (utils.py:139-191);
 *   NRT_NEAREST: int32(round_half_even(loc)) THEN clip (utils.py:196-197).
 *   has_fill: out = out*(!oob) + oob*fill with oob on the UNCLIPPED loc, strict (utils.py:206-213).
 * ------------------------------------------------------------------------------------- */
NRT_API int nrt_interpn_f32(const float* vol, const int32_t* vol_shape, int D, int C,
                    const float* loc, int64_t n_out, int method, int has_fill, float fill,
                    float* out, void* stream);

/* interpn whose sample grid has the volume's own spatial shape (D = 3): loc [S0,S1,S2,3]
 * -> out [S0,S1,S2,C].  Same results as nrt_interpn_f32; samples that stay within `halo`
 * voxels (plus a coherent shift) of their own grid position are served from the TMA-staged
 * shared-memory tiles of the warp kernel.  This is the shape voxelmorph's transform() hands
 * to neurite.utils.interpn (utils.py:73-220). */
NRT_API int nrt_interpn_grid_f32(const float* vol, const float* loc, float* out, const int32_t* shape,
                         int C, int method, int has_fill, float fill, int halo, void* stream);

/* ---------------------------------------------------------------------------------------
 * warp -- replaces voxelmorph.layers.SpatialTransformer on a dense shift (call sites
 * neurite/tf/models.py:806-807, 1157-1159): out[b] = interpn(vol[b], ndgrid + flow[b]).
 * The identity grid is generated in registers (no loc tensor).
 *   vol  [B, src_n0, S_1.., C]  the planes [src_z0, src_z0+src_n0) of a volume whose full
 *                               extent along spatial axis 0 is full_s0 (slab sharding;
 *                               pass src_z0=0, src_n0=full_s0 for a whole volume)
 *   flow [B, out_n0, S_1.., D]  shifts for output planes [out_z0, out_z0+out_n0)
 *   out  [B, out_n0, S_1.., C]
 *   shape = {full_s0, S_1, S_2} (D entries).  Coordinates are clipped against the FULL
 *   volume; a corner that falls outside the resident source planes sets *err_flag (device
 *   int32, may be null) and reads the nearest resident plane.
 *   halo: expected max |flow| in voxels (tiling hint for the shared-memory path only;
 *   results do not depend on it).  <=0 selects the default (3).
 * ------------------------------------------------------------------------------------- */
NRT_API int nrt_warp_f32(const float* vol, const float* flow, float* out, int B,
                 const int32_t* shape, int D, int C, int method, int has_fill, float fill,
                 int src_z0, int src_n0, int out_z0, int out_n0, int halo,
                 int32_t* err_flag, void* stream);
/* The same warp on batch items that are not densely packed: *_batch_stride = elements between consecutive batch
 * items of vol / flow / out (0 = dense).  This is what lets a z-slab-sharded warp (SURVEY.md 8e; call sites
 * neurite/tf/models.py:806-807) produce the INTERIOR planes of a slab from the rank's own planes while the halo
 * planes of the neighbours are still in flight, and the boundary planes afterwards, all inside one [B, planes, ...]
 * buffer: plane sub-ranges of a batched slab are strided in the batch dimension. */
NRT_API int nrt_warp_strided_f32(const float* vol, const float* flow, float* out, int B,
                 const int32_t* shape, int D, int C, int method, int has_fill, float fill,
                 int src_z0, int src_n0, int out_z0, int out_n0, int halo,
                 int32_t* err_flag, int64_t vol_batch_stride, int64_t flow_batch_stride,
                 int64_t out_batch_stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * resize -- replaces neurite/tf/utils/utils.py:223-265 (resize/zoom) and the per-batch
 * map of neurite/tf/layers.py:154-181 (Resize.call).  Sample positions come from an
 * in-kernel fp32 linspace(0, S_d-1, M_d) (endpoints exact, interior delta*i), no grid tensor.
 *   vol [B, S.., C] -> out [B, M.., C];  out planes [out_z0, out_z0+out_n0) of axis 0 are
 *   produced (slab sharding; out points at the first produced plane).
 * ------------------------------------------------------------------------------------- */
NRT_API int nrt_resize_f32(const float* vol, float* out, int B, const int32_t* in_shape,
                   const int32_t* out_shape, int D, int C, int method,
                   int out_z0, int out_n0, void* stream);

/* ---------------------------------------------------------------------------------------
 * Dice -- replaces neurite/tf/metrics.py:415-482 (Dice.dice) after batch_channel_flatten.
 *   y_true, y_pred [B, V, L] fp32.  One pass produces sums[b,l,{0,1,2}] =
 *   {sum t*p, sum t*t, sum p*p} over voxels [v0, v0+nv) of every batch item (voxel-range
 *   sharding: all-reduce `sums` across ranks, then finalize), and ORs bit0 into *flag if
 *   any element of t or p is outside [0,1] (or NaN) when check_limits != 0
 *   (metrics.py:439-444).  workspace: device scratch of nrt_dice_workspace_bytes(B,L).
 *   normalize != 0 divides each voxel's labels by their sum first (divide_no_nan, :434-436).
 * ------------------------------------------------------------------------------------- */
NRT_API int64_t nrt_dice_workspace_bytes(int B, int L);
NRT_API int nrt_dice_sums_f32(const float* y_true, const float* y_pred, int B, int64_t V, int L,
                      int64_t v0, int64_t nv, int normalize, int check_limits,
                      float* sums, int32_t* flag, void* workspace, int64_t workspace_bytes,
                      void* stream);
/* hard Dice on label maps (metrics.py:450-468 without materialising one-hot):
 *   t_lab, p_lab [B, V] int32; sums as above (counts).  Labels outside [0,L) count nowhere. */
NRT_API int nrt_dice_label_sums_i32(const int32_t* t_lab, const int32_t* p_lab, int B, int64_t V, int L,
                            int64_t v0, int64_t nv, float* sums, void* workspace,
                            int64_t workspace_bytes, void* stream);
/* argmax over the last axis (first max wins, like tf.argmax): x [n, L] -> idx [n] int32 */
NRT_API int nrt_argmax_f32(const float* x, int64_t n, int L, int32_t* idx, void* stream);
/* dice[b,l] = laplace>0 ? (2*tp+eps)/(tt+pp+eps) : divide_no_nan(2*tp, tt+pp)  (:476-482) */
NRT_API int nrt_dice_finalize_f32(const float* sums, int B, int L, float laplace, float* dice,
                          void* stream);

/* ---------------------------------------------------------------------------------------
 * Categorical cross-entropy -- replaces neurite/tf/metrics.py:640-650 plus the Keras
 * CategoricalCrossentropy arithmetic underneath (third party): t *= w_label;
 * [label smoothing]; p /= sum_c p; p = clip(p, 1e-7, 1-1e-7); l = -sum_c t*log p
 * (from_logits: l = -sum_c t*log_softmax(p)); l *= sample_weight.
 *   y_true, y_pred [n, C]; label_w [C] or null; sample_w [n] or null;
 *   per_elem [n] or null (reduction 'none'); sum_out [1] (fp32 sum of l over the n rows;
 *   the caller divides by the global n for 'sum_over_batch_size').
 *   workspace: nrt_cce_workspace_bytes().
 * ------------------------------------------------------------------------------------- */
NRT_API int64_t nrt_cce_workspace_bytes(void);
NRT_API int nrt_cce_f32(const float* y_true, const float* y_pred, const float* label_w,
                const float* sample_w, int64_t n, int C, int from_logits, float label_smoothing,
                float* per_elem, float* sum_out, void* workspace, int64_t workspace_bytes,
                void* stream);

/* ---------------------------------------------------------------------------------------
 * LocallyConnected3D, implementation 1 -- replaces neurite/tf/layers.py:1072-1102 (call)
 * and :1126-1197 (local_conv): out[b,p,f] = act(sum_j patch[b,p,j]*kernel[p,j,f] + bias[p,f]).
 *   x      [B, I0, I1, I2, Cin]  (channels-last storage)
 *   kernel [P, F, Cout], P = O0*O1*O2 row-major, F = k0*k1*k2*Cin (layers.py:974-977)
 *   bias   [O0, O1, O2, Cout] or null (layers.py:1034-1040)
 *   out    [B, p_count, Cout] for output positions [p0, p0+p_count) (position sharding:
 *          kernel/bias/out point at position p0 of the rank's shard)
 *   feature_order 0: j = ((i0*k1+i1)*k2+i2)*Cin + c   (data_format channels_last)
 *                 1: j = ((c*k0+i0)*k1+i1)*k2+i2     (kernel trained channels_first)
 *   'valid' padding only (layers.py:934-936).
 * ------------------------------------------------------------------------------------- */
NRT_API int nrt_lc3d_fwd_f32(const float* x, const float* kernel, const float* bias, float* out,
                     int B, const int32_t* in_shape, int Cin, int Cout,
                     const int32_t* ksize, const int32_t* strides, int feature_order,
                     int activation, int64_t p0, int64_t p_count, void* stream);

/* ---------------------------------------------------------------------------------------
 * Gradients (SURVEY.md 8f item 1).  The reference obtains them from TensorFlow autodiff of
 * the op graphs cited above; these entry points are that graph differentiated by hand
 * (floor/round: zero gradient; clip_by_value: passes on the closed interval; gather:
 * scatter-add).  grad_vol buffers are ACCUMULATED into (atomics) -- zero them first.
 * Whole volumes only (no slab arguments).
 * ------------------------------------------------------------------------------------- */
/* backward of nrt_warp_f32: grad_out [B,S..,C] -> grad_vol [B,S..,C] (may be null),
 * grad_flow [B,S..,D] (may be null; zeros for NRT_NEAREST) */
NRT_API int nrt_warp_bwd_f32(const float* vol, const float* flow, const float* grad_out, float* grad_vol,
                     float* grad_flow, int B, const int32_t* shape, int D, int C, int method,
                     int has_fill, void* stream);
/* backward of nrt_interpn_f32: grad_out [n_out,C] -> grad_vol [S..,C], grad_loc [n_out,D] */
NRT_API int nrt_interpn_bwd_f32(const float* vol, const int32_t* vol_shape, int D, int C, const float* loc,
                        int64_t n_out, int method, int has_fill, const float* grad_out,
                        float* grad_vol, float* grad_loc, void* stream);
/* backward of nrt_resize_f32 (sample positions are constants): grad_out [B,M..,C] -> grad_vol [B,S..,C] */
NRT_API int nrt_resize_bwd_f32(const float* grad_out, float* grad_vol, int B, const int32_t* in_shape,
                       const int32_t* out_shape, int D, int C, int method, void* stream);
/* backward of Dice.dice: given sums [B,L,3] from nrt_dice_sums_f32 and grad_dice [B,L],
 * grad_pred = a*t - c*p, grad_true = a*p - c*t with a = 2G/(bot+eps), c = 2G(top+eps)/(bot+eps)^2
 * (both 0 where bot == 0 and eps == 0: divide_no_nan).  Either output may be null. */
NRT_API int nrt_dice_bwd_f32(const float* y_true, const float* y_pred, const float* sums,
                     const float* grad_dice, int B, int64_t V, int L, float laplace,
                     float* grad_true, float* grad_pred, void* stream);
/* backward of nrt_cce_f32 wrt y_pred: upstream = scale * (*grad_scalar if non-null) *
 * (grad_per_elem[r] if non-null) * sample_w[r]. */
NRT_API int nrt_cce_bwd_f32(const float* y_true, const float* y_pred, const float* label_w,
                    const float* sample_w, int64_t n, int C, int from_logits, float label_smoothing,
                    const float* grad_scalar, float scale, const float* grad_per_elem,
                    float* grad_pred, void* stream);

/* backward of nrt_lc3d_fwd_f32 (linear activation; apply the activation's derivative to
 * grad_out first): grad_out [B,p_count,Cout] -> grad_kernel [p_count,F,Cout] (overwritten),
 * grad_x [B,I0,I1,I2,Cin] (ACCUMULATED: overlapping patches, zero it first).  Either may be
 * null.  grad_bias[p,f] = sum_b grad_out[b,p,f] is left to the caller. */
NRT_API int nrt_lc3d_bwd_f32(const float* x, const float* kernel, const float* grad_out, float* grad_x,
                     float* grad_kernel, int B, const int32_t* in_shape, int Cin, int Cout,
                     const int32_t* ksize, const int32_t* strides, int feature_order,
                     int64_t p0, int64_t p_count, void* stream);

/* ---- mutual information (SURVEY.md 8f-3; neurite/tf/metrics.py:41-336, utils.py:1099-1172) ----
 * Two operands over nv voxels of each of B items.  An operand is either
 *   quant = 1: an intensity image, element (b, v, c) at p[b*batch_stride + v*vox_stride + c],
 *              soft-quantised in registers: w[bin] = exp(-alpha * (clip(x, min_clip, max_clip) - centers[bin])^2)
 *              (soft_quantize, utils.py:1157-1171); C channels are processed independently
 *              (MutualInformation.channelwise, metrics.py:185-225);
 *   quant = 0: a probability / similarity map, element (b, v, bin) at p[b*batch_stride + v*vox_stride + bin]
 *              (MutualInformation.maps, metrics.py:227-292); requires C == 1.
 * stats[(b*C + c)][nbx*nby + nbx + nby] = joint sums  sum_v wx[i]*wy[j]  (row-major i, j), then
 * sum_v wx[i], then sum_v wy[j]  -- the three reductions metrics.py:272-283 need.  Voxel-range
 * sharding across GPUs: every rank passes its own voxel slab (pointer offset, nv) and the stats
 * are summed (one all-reduce) before nrt_mi_finalize_f32.  *flag is set to 1 if a map value is
 * negative (tf.debugging.assert_non_negative, metrics.py:262-263).  bins <= 64; bins <= 32 run on
 * the tensor cores (3xTF32 mma).  workspace: nrt_mi_workspace_bytes(B*C, nbx, nby). */
NRT_API int64_t nrt_mi_workspace_bytes(int items, int nbx, int nby);
NRT_API int nrt_mi_hist_f32(const float* x, int64_t x_batch_stride, int64_t x_vox_stride, int x_quant, int nbx,
                    const float* x_centers, const float* y, int64_t y_batch_stride, int64_t y_vox_stride,
                    int y_quant, int nby, const float* y_centers, int B, int C, int64_t nv, float alpha,
                    float min_clip, float max_clip, float* stats, int32_t* flag, void* workspace,
                    int64_t workspace_bytes, void* stream);
/* metrics.py:265-292 on the sums:  pxy = h/(sum h + eps), px = sx/(sum sx + eps), py likewise,
 * mi[item] = sum_ij pxy * log(pxy / (px*py + eps) + eps);  eps = K.epsilon() = 1e-7. */
NRT_API int nrt_mi_finalize_f32(const float* stats, int items, int nbx, int nby, float eps, float* mi, void* stream);
/* ---- gradient of the mutual information (TF autodiff through metrics.py:227-292 and
 * utils.py:1099-1172).  nrt_mi_finalize_bwd_f32: gstats[item] = grad_mi[item] * d mi / d stats[item]
 * (same [nbx*nby + nbx + nby] layout).  nrt_mi_bwd_f32: one pass over the voxels (operands as in
 * nrt_mi_hist_f32, bins <= 32) writing grad_x / grad_y in the operands' own layout (either may be
 * null); for a quantised operand the clip passes the gradient on [min_clip, max_clip].  If
 * `dcenters` ([2][34] floats) is non-null it receives, per operand, d L / d centre[i] (i < nb)
 * followed by the number of elements equal to centre[0] and to centre[nb-1]; when the centres are
 * linspace(min, max) of the tensor, nrt_mi_minmax_bwd_f32 then adds the share of every element equal
 * to the minimum / maximum to grad_x (TF's reduce_min / reduce_max gradient).  With voxel-range
 * sharding, sum `dcenters` over the ranks first. */
NRT_API int nrt_mi_finalize_bwd_f32(const float* stats, const float* grad_mi, int items, int nbx, int nby, float eps,
                            float* gstats, void* stream);
NRT_API int64_t nrt_mi_bwd_workspace_bytes(int items);
NRT_API int nrt_mi_bwd_f32(const float* x, int64_t x_batch_stride, int64_t x_vox_stride, int x_quant, int nbx,
                   const float* x_centers, const float* y, int64_t y_batch_stride, int64_t y_vox_stride,
                   int y_quant, int nby, const float* y_centers, int B, int C, int64_t nv, float alpha,
                   float min_clip, float max_clip, const float* gstats, float* grad_x, float* grad_y,
                   float* dcenters, void* workspace, int64_t workspace_bytes, void* stream);
NRT_API int nrt_mi_minmax_bwd_f32(const float* x, int64_t n, const float* minmax, const float* dcenters, int nb,
                          float* grad_x, void* stream);
/* centers = tf.linspace(minmax[0], minmax[1], nb) in fp32 (utils.py:1153), all on the device; minmax = {min(x),
 * max(x)} (K.min / K.max, utils.py:1151-1152) is nrt_item_stats_f32 with items = 1 and NRT_STAT_MINMAX. */
NRT_API int nrt_mi_bin_centers_f32(const float* minmax, int nb, float* centers, void* stream);
/* soft_quantize as a tensor op (utils.py:1099-1172): out[e*nb + b], e < n. */
NRT_API int nrt_soft_quantize_f32(const float* x, int64_t n, const float* centers, int nb, float alpha, float min_clip,
                          float max_clip, int return_log, float* out, void* stream);

/* ---- separable convolution pass / GaussianBlur / Subsample (SURVEY.md 8f-4) -------------------
 * One 1-D cross-correlation pass of separable_conv (utils.py:665-751): x viewed as
 * [outer, L, inner] -> out [outer, L_out, inner],
 *   out[o, l, i] = sum_j kernel[j] * x[o, l*stride - pad_before + j*dilation, i]   (zero outside [0, L)).
 * The caller derives pad_before / L_out from TF's 'SAME' / 'VALID' rules.  kernel is a device
 * pointer ([K]).  x and out must not alias. */
NRT_API int nrt_sepconv_axis_f32(const float* x, float* out, int64_t outer, int64_t L, int64_t inner, const float* kernel,
                         int K, int stride, int dilation, int pad_before, int64_t L_out, void* stream);
/* out[o, l, i] = x[o, index[l], i]: tf.gather along an axis (subsample_axis, utils.py:818-823). */
NRT_API int nrt_gather_axis_f32(const float* x, const int32_t* index, float* out, int64_t outer, int64_t L, int64_t inner,
                        int64_t L_out, void* stream);

/* ---- noise fields: PerlinNoise / GaussianNoise (layers.py:2305-2508, augment.py:65-218) ----------------------
 * A counter-based Philox4x32-10 stream: element i of a draw with `key` depends on (key, i) only (nrt_noise.cu
 * documents the integer -> float conversion and the Box-Muller arithmetic).  Draws hold at most 2^31-1 elements.
 * out[i] = lo + (hi - lo) * u_i, u_i in (0, 1]. */
NRT_API int nrt_philox_uniform_f32(uint64_t key, int64_t n, float lo, float hi, float* out, void* stream);
/* out[i] = z_i * sd[t(i)] * (*sd_scale if non-null) (+ x[i] if x is non-null), z_i standard normal.  shape[ndim]
 * is the draw's row-major shape (ndim <= 5); the SD table sd has the row-major shape sd_shape[ndim], each extent
 * equal to shape's or 1 (broadcast).  x may be null and must not alias out. */
NRT_API int nrt_philox_normal_f32(uint64_t key, const int32_t* shape, const int32_t* sd_shape, int ndim, const float* sd,
                          const float* sd_scale, const float* x, float* out, void* stream);
/* Per-item reductions of x [items, n], deterministic (fixed-order block partials; the grid depends on (items, n)
 * only).  SD: out[item] = population SD (fp64 sums of d = x - x[item, 0]; tf.math.reduce_std); MAX: max x;
 * ABSMAX: max |x|; MINMAX: out[2 item] = min x, out[2 item + 1] = max x.  The extrema skip NaNs (fminf / fmaxf).
 * workspace: nrt_item_stats_workspace_bytes(items, n). */
NRT_API int64_t nrt_item_stats_workspace_bytes(int items, int64_t n);
NRT_API int nrt_item_stats_f32(const float* x, int items, int64_t n, int kind, float* out, void* workspace,
                       int64_t workspace_bytes, void* stream);
/* Mean over Perlin levels: x [L, G, m] -> out [G, m],
 *   out[g, i] = (sum_l x[l, g, i] * divide_no_nan(before[l*G + g], after[l*G + g])) / L   (levels in order). */
NRT_API int nrt_level_combine_f32(const float* x, int L, int G, int64_t m, const float* before, const float* after,
                          float* out, void* stream);
/* GaussianNoise fused with the generator's background clearing (models.py:1219-1231), x and out [B, V, C]:
 *   out[i] = (x[i] + z_i * (sd[b * C + c] * *sd_scale)) * (label(b, v) == 0 && bg_u[b] < zero_background ? 0 : 1)
 * with z_i the normals of nrt_philox_normal_f32 for the same key and shape [B, V, C], bit for bit.  label(b, v) is
 * int32(labels[b * V + v]) inside the crop window of nrt_labels_to_image_f32, 0 outside. */
NRT_API int nrt_philox_normal_background_f32(uint64_t key, int B, int64_t V, int C, const float* sd,
                          const float* sd_scale, const float* x, const float* labels, int64_t crop_L,
                          int64_t crop_inner, int64_t crop_lo, int64_t crop_hi, const float* bg_u,
                          float zero_background, float* out, void* stream);

/* ---- label-to-image synthesis: labels_to_image_new (models.py:1162-1282), RandomCrop (layers.py:446-519) ------
 * labels [B, V] fp32 holds the warped label map; a voxel's label is int32(trunc(x)).  The crop window keeps the
 * voxels v with (v / crop_inner) % crop_L in [crop_lo, crop_hi) and sets the others' label to 0; (1, 1, 0, 1)
 * keeps all.  A LUT lookup outside [0, nlut) gives 0 (TF's GPU gather).
 * Image: idx = gen_lut[label]; mean = u[b, c, idx] * (mean_max[c, idx] - mean_min[c, idx]) + mean_min[c, idx]
 * (mean_min / mean_max [C, N]);
 * image[b, v, c] = mean (* f, f = bias[b, v, c], expf'd when apply_exp), each op rounded once.  mean_out and
 * bias_out (may be null; need bias) receive mean and f.  *absmax = max |image| over the whole batch (device
 * scalar, deterministic).  workspace: nrt_labels_to_image_workspace_bytes(). */
NRT_API int64_t nrt_labels_to_image_workspace_bytes(void);
NRT_API int nrt_labels_to_image_f32(const float* labels, int B, int64_t V, int C, int64_t crop_L, int64_t crop_inner,
                          int64_t crop_lo, int64_t crop_hi, const int32_t* gen_lut, int nlut, int N,
                          const float* u, const float* mean_min, const float* mean_max, const float* bias,
                          int apply_exp, float* image, float* mean_out, float* bias_out, float* absmax,
                          void* workspace, int64_t workspace_bytes, void* stream);
/* x [items, n] with n = V * C -> out: y = x; with mnmx (the NRT_STAT_MINMAX output of nrt_item_stats_f32),
 * y = div_no_nan(y - mn, mx - mn); with gamma_u [items, C], y = powf(y, gamma_u[item, c] * (gamma_hi - gamma_lo) +
 * gamma_lo).  out must not alias x. */
NRT_API int nrt_norm_gamma_f32(const float* x, int items, int64_t n, int C, const float* mnmx, const float* gamma_u,
                          float gamma_lo, float gamma_hi, float* out, void* stream);
/* Output label map: l = crop(label), then l = lut[l] when lut is non-null.  _f32 writes the one-hot out [B, V, M]
 * (all-zero row when l is outside [0, M)); _i32 writes l to out [B, V]. */
NRT_API int nrt_label_map_f32(const float* labels, int B, int64_t V, int64_t crop_L, int64_t crop_inner,
                          int64_t crop_lo, int64_t crop_hi, const int32_t* lut, int nlut, int M, float* out,
                          void* stream);
NRT_API int nrt_label_map_i32(const float* labels, int B, int64_t V, int64_t crop_L, int64_t crop_inner,
                          int64_t crop_lo, int64_t crop_hi, const int32_t* lut, int nlut, int32_t* out, void* stream);
/* out[o, l, i] = x[o, l, i] * (lo <= l < hi) on [outer, L, inner] (RandomCrop's mask); out must not alias x. */
NRT_API int nrt_crop_window_f32(const float* x, int64_t outer, int64_t L, int64_t inner, int64_t lo, int64_t hi,
                          float* out, void* stream);
NRT_API int nrt_crop_window_i32(const int32_t* x, int64_t outer, int64_t L, int64_t inner, int64_t lo, int64_t hi,
                          int32_t* out, void* stream);
/* The generator's label warp (models.py:1130-1160) in one pass: labels [B, *in_shape, 1] fp32, mats [B, N, N+1] fp32
 * (one affine per item), def [B, *out_shape, N] fp32 or null -> out [B, *out_shape, 1], N = 2 or 3.  With the dense
 * shift s_i(c) = ((M_i0 c_0 + M_i1 c_1) + M_i2 c_2) + M_iN - c_i at integer out-grid points c, t = s(x) without def
 * and t = def(x) + interpn_linear(s, x + def(x)) with it; out = the nearest sample of the labels at x + t, 0 outside
 * the in grid.  Every op is rounded once: bit for bit AffineToDenseShift, ComposeTransform and the nearest
 * SpatialTransformer with fill 0. */
NRT_API int nrt_warp_labels_affine_f32(const float* labels, const float* mats, const float* def, float* out, int B,
                          int N, const int32_t* in_shape, const int32_t* out_shape, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEURITE_B200_H_ */
