/*
 * b2second.h -- C ABI of libb2second.so: the H100 (sm_90a) implementation of the native layer that
 * second.pytorch reaches through the external `spconv` 1.x package on its LiDAR-inference hot path.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter is marked "host";
 *   - all counts that depend on data live in device memory (`*_dev`); no entry point synchronises,
 *     allocates, or keeps global mutable state; the caller owns all memory and passes workspaces;
 *   - `stream` is the caller's cudaStream_t (as void*), e.g. torch.cuda.current_stream().cuda_stream;
 *   - return 0 on success, negative on error; b2s_last_error() (thread-local) gives the message;
 *   - data-dependent overflow of a caller-sized buffer never writes out of bounds: it raises bit(s)
 *     in the caller's `status_dev` word (B2S_STATUS_*), which the caller reads when it next syncs;
 *   - coordinates are int32 rows (b, z, y, x); features are fp32 row-major [rows, channels].
 *
 * What each entry point replaces (paths relative to the reference root; the spconv symbols are the
 * ones those call sites bind -- spconv itself is not vendored in the reference):
 *
 *   b2s_voxelize        spconv.utils.VoxelGeneratorV2.generate / generate_multi_gpu
 *                       (second/builder/voxel_builder.py:23-32, second/data/preprocess.py:303-315)
 *                       + fused SimpleVoxel / SimpleVoxelRadius mean
 *                       (second/pytorch/models/voxel_encoder.py:206-255)
 *   b2s_hash_build,
 *   b2s_rulebook_subm,
 *   b2s_rulebook_conv   torch.ops.spconv.get_indice_pairs as used by spconv.SubMConv3d / SparseConv3d
 *                       (second/pytorch/models/middle.py:146-189)
 *   b2s_sparse_conv     torch.ops.spconv.indice_conv (+ the BatchNorm1d/ReLU that always follow,
 *                       middle.py:146-191, folded into scale/shift/relu)
 *   b2s_to_bev          spconv.SparseConvTensor.dense() + view (middle.py:206-209) and
 *                       PointPillarsScatter.forward (second/pytorch/models/pointpillars.py:444-476)
 *   b2s_pfn             PillarFeatureNet.forward (pointpillars.py:203-237, single PFNLayer :51-65)
 *   b2s_decode_filter   box_coder.decode_torch + sigmoid + score threshold
 *                       (second/pytorch/models/voxelnet.py:413-414,444,560-576,
 *                        second/pytorch/core/box_torch_ops.py:56-102)
 *   b2s_nms             torch.topk + spconv.utils.rotate_non_max_suppression_cpu /
 *                       spconv.utils.non_max_suppression (box_torch_ops.py:454-515,
 *                       second/core/non_max_suppression/nms_cpu.py:20-31, nms_gpu.py:10-19)
 *                       + direction / range epilogue (voxelnet.py:598-628)
 *   b2s_nms_aligned_host, b2s_nms_rotated_host
 *                       the numpy-facing spconv.utils.non_max_suppression /
 *                       rotate_non_max_suppression_cpu signatures (host arrays in, keep list out)
 */
#ifndef B2SECOND_H_
#define B2SECOND_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 200

/* status bits raised in *status_dev */
#define B2S_STATUS_VOXEL_OVERFLOW 1u   /* more voxels than max_voxels (extra voxels dropped, as spconv) */
#define B2S_STATUS_ROWS_OVERFLOW 2u    /* strided conv produced more rows than cap_out (rows dropped)   */
#define B2S_STATUS_HASH_FULL 4u        /* hash table too small                                            */
#define B2S_STATUS_CAND_OVERFLOW 8u    /* more score-threshold survivors than cand_cap (lowest dropped)  */
#define B2S_STATUS_F16_RANGE 16u       /* an activation left the fp16 range (|x| > 65504) on the tensor-core path;
                                          it was clamped -- results are not fp32-grade for that frame batch      */

/* IEEE binary16 bit pattern (the tensor-core kernels' operand planes; torch.float16 storage) */
typedef uint16_t b2s_half;

int b2s_version(void);
const char *b2s_last_error(void);

/* ---- on-GPU input path in front of the voxelizer (SURVEY.md §8(f)1) ------------------------------- */
/* One NuScenes sweep -> rows [x', y', z', time_lag] of the merged cloud (second/data/nuscenes_dataset.py:166-185):
 * (x', y', z') = float32(float32(p @ R^T, computed in float64) + t), rotation_host row-major [3,3] / translation_host [3]
 * float64 (NULL rotation: the key-frame sweep, copied as is).  points_in [P, feat_in] (x, y, z first); out [P, 4],
 * 16-byte aligned (pass the merged buffer advanced to the sweep's first row). */
int b2s_transform_sweep(const float *points_in, int num_points, int feat_in, const double *rotation_host,
                        const double *translation_host, float time_lag, float *out, void *stream);

/* Keep the points strictly inside a convex polytope, in input order: inside <=> a x + b y + c z + d < 0 (float64)
 * for every plane (a, b, c, d) of planes_host [num_planes, 4] -- the KITTI camera-frustum crop
 * remove_outside_points (second/core/box_np_ops.py:682-693) with the plane equations of
 * surface_equ_3d_jitv2 (second/core/geometry.py:332-355).  The kept points of this frame are written to
 * out_points[offsets_dev[0] ...] (rows of num_feat floats) and offsets_dev[1] = offsets_dev[0] + kept: calling it for
 * frames 0..B-1 with offsets_dev + b fills the voxelizer's point buffer and frame_offsets without a host sync.
 * Rows that would pass out_cap_rows are dropped (B2S_STATUS_ROWS_OVERFLOW). */
size_t b2s_crop_workspace_bytes(int num_points);
int b2s_crop_convex(const float *points, int num_points, int num_feat, const double *planes_host, int num_planes,
                    float *out_points, int out_cap_rows, int *offsets_dev, void *workspace, size_t workspace_bytes,
                    unsigned *status_dev, void *stream);

/* ---- voxelizer -------------------------------------------------------------------------------- */
/* VFE modes fused into the voxelizer */
#define B2S_VFE_NONE 0
#define B2S_VFE_MEAN 1        /* SimpleVoxel: mean of the first num_features point features          */
#define B2S_VFE_MEAN_RADIUS 2 /* SimpleVoxelRadius: [norm(mean xy), mean[2:num_features]]            */

size_t b2s_voxelize_workspace_bytes(int num_points, int batch, int max_voxels, int max_points);
int b2s_voxelize_hash_capacity(int num_points);

/* points [P,F] fp32 for `batch` frames stored back to back; frame_offsets_dev [batch+1] int32 (may be
 * NULL when batch==1; when given, frame_offsets_dev[batch] is the live point count and num_points is
 * only the buffer capacity -- points beyond it are ignored).  Frame-major first-come voxel ids, at most max_voxels per frame; rows of all
 * frames are compacted back to back (frame 0 first), exactly the layout merge_second_batch builds
 * (second/data/preprocess.py:21-55).
 * outputs (row capacity = batch*max_voxels):
 *   coors [cap,4] (b,z,y,x); num_points_per_voxel [cap]; point_slots [cap,T] point indices (-1 pad),
 *   voxels [cap,T,F] zero padded (may be NULL); vfe_out [cap,vfe_channels] (NULL if vfe_mode==NONE);
 *   num_voxels_dev [1+batch]: total then per-frame counts;
 *   hash_keys [hash_cap] u64 / hash_vals [hash_cap] i32: coordinate -> row locator of the result. */
int b2s_voxelize(const float *points, const int *frame_offsets_dev, int num_points, int num_feat,
                 int batch, const float *range_lo /*host[3] xyz*/, const float *voxel_size /*host[3]*/,
                 const int *grid /*host[3] xyz*/, int max_points, int max_voxels, int *coors,
                 int *num_points_per_voxel, int *point_slots, float *voxels, int vfe_mode,
                 int vfe_num_features, float *vfe_out, int *num_voxels_dev,
                 unsigned long long *hash_keys, int *hash_vals, int hash_cap,
                 int hash_key_depth /*D of the flat (b,z,y,x) hash key = spatial_shape[0] of the tensor that will
                                      look rows up (SECOND: grid_z + 1, middle.py:139); 0 = grid z*/,
                 void *workspace, size_t workspace_bytes, unsigned *status_dev, void *stream);

/* SimpleVoxel / SimpleVoxelRadius (second/pytorch/models/voxel_encoder.py:220-225,246-255) over voxels that arrive
 * already gathered -- the reference's own example dict: voxels [rows, T, F] zero padded, num_points_per_voxel
 * [rows]; rows = *num_rows_dev.  vfe_mode B2S_VFE_MEAN -> vfe_out [rows, nf]; B2S_VFE_MEAN_RADIUS -> [rows, nf-1]. */
int b2s_vfe_mean(const float *voxels, const int *num_points_per_voxel, const int *num_rows_dev, int cap_rows, int T,
                 int F, int vfe_mode, int vfe_num_features, float *vfe_out, void *stream);

/* ---- rulebook --------------------------------------------------------------------------------- */
/* coordinate -> row hash over `shape` (D,H,W).  hash_cap must be a power of two >= 2*cap_rows. */
int b2s_hash_build(const int *coors, const int *num_rows_dev, int cap_rows, const int *shape /*host[3]*/,
                   unsigned long long *hash_keys, int *hash_vals, int hash_cap, unsigned *status_dev,
                   void *stream);

/* submanifold conv rulebook: nbr[row][k] = input row at coor + (k - k//2)*dil, or -1.
 * k index row-major over (kz,ky,kx); K = kz*ky*kx.
 * row_mask (optional, all three rulebook builders): [rows] bit k = nbr[row][k] exists -- what b2s_sparse_tile_plan needs,
 * written while the table is built so that the plan does not have to read the table again. */
int b2s_rulebook_subm(const int *coors, const int *num_rows_dev, int cap_rows, const int *shape,
                      const int *ksize /*host[3]*/, const int *dilation /*host[3]*/,
                      const unsigned long long *hash_keys, const int *hash_vals, int hash_cap,
                      int *nbr /*[cap_rows,K]*/, unsigned *row_mask /*[cap_rows] or NULL*/, void *stream);

size_t b2s_rulebook_conv_workspace_bytes(int batch, const int *out_shape /*host[3]*/);
/* strided ("regular") sparse conv rulebook.  Output rows are emitted sorted ascending by flat
 * (b,z,y,x) key.  out_shape must be (in + 2p - d(k-1) - 1)/s + 1 per dim.
 * Builds the out-coordinate hash as well (hash_cap_out power of two >= 2*cap_out). */
int b2s_rulebook_conv(const int *coors_in, const int *num_in_dev, int cap_in, int batch,
                      const int *in_shape, const int *out_shape, const int *ksize, const int *stride,
                      const int *padding, const int *dilation, const unsigned long long *hash_keys_in,
                      const int *hash_vals_in, int hash_cap_in, int *coors_out /*[cap_out,4]*/,
                      int *num_out_dev, int cap_out, int *nbr /*[cap_out,K]*/,
                      unsigned long long *hash_keys_out, int *hash_vals_out, int hash_cap_out,
                      void *workspace, size_t workspace_bytes, unsigned *row_mask /*[cap_out] or NULL*/,
                      unsigned *status_dev, void *stream);

/* SubM rulebook of the level b2s_rulebook_conv has JUST produced, read off the occupancy structure that call left in
 * `workspace` (same batch / shape, nothing else run on the workspace in between): coordinate -> row is a bit test +
 * popcount rank, no hash table.  Pass hash_keys_out = hash_vals_out = NULL to b2s_rulebook_conv when every SubM of
 * the produced level is built this way.  nbr as b2s_rulebook_subm. */
int b2s_rulebook_subm_ranked(const int *coors, const int *num_rows_dev, int cap_rows, int batch, const int *shape,
                             const int *ksize, const int *dilation, const void *workspace, size_t workspace_bytes,
                             int *nbr, unsigned *row_mask /*[cap_rows] or NULL*/, void *stream);

/* pair-list view of a neighbour table (spconv's indice_pairs [K,2,L] + indice_pair_num [K]) --
 * only for parity checks / API completeness; the conv kernels consume `nbr` directly. */
int b2s_rulebook_pairs(const int *nbr, const int *num_out_dev, int cap_out, int K, int L,
                       int *indice_pairs /*[K,2,L] prefilled -1*/, int *indice_pair_num /*[K] zeroed*/,
                       void *stream);

/* ---- sparse convolution ------------------------------------------------------------------------ */
/* out[o,:] = act( (sum_k W[k]^T in[nbr[o,k],:]) * scale + shift ),  W = [K,Cin,Cout] fp32
 * (the reference's weight [kD,kH,kW,Cin,Cout] viewed flat).  scale/shift may be NULL (identity);
 * a conv bias is passed as shift with scale NULL.  Accumulation order: k ascending, fp32. */
int b2s_sparse_conv(const float *feat_in, int cin, const float *weight, const int *nbr, int K,
                    const int *num_out_dev, int cap_out, const float *scale, const float *shift,
                    int relu, float *feat_out, int cout, void *stream);

/* same contraction on the tensor pipe (wgmma f16, 3xF16 hi/lo split, fp32-grade): Cin in {8,16,32,64}, Cout in
 * {16,32,64}, K <= 27 (b2s_sparse_conv_tc_supported).  Every fp32 operand x travels as two fp16 planes hi = fp16(x),
 * lo = fp16(x - hi); per K step the kernel issues A_hi*W_hi + A_hi*W_lo + A_lo*W_hi with fp32 accumulation.
 *   feat_hi/lo  rows of in_stride halves (>= Cin, multiple of 8; e.g. interleaved [row][hi Cin | lo Cin] with
 *               feat_lo = feat_hi + Cin, in_stride = 2*Cin); a 3/4-feature input layer is zero-padded to Cin = 8;
 *   w_hi/lo     [K, Cout, 64] for Cin = 64; for Cin < 64 the 64/Cin consecutive kernel offsets that share one
 *               128-byte K block are packed side by side: [ceil(K/(64/Cin)), Cout, 64], column = offset_in_pack*Cin +
 *               cin, zero columns past K.  Weights may be pre-scaled by a power of two folded into `scale`;
 *   out_hi/lo   rows of out_stride halves; out_lo NULL -> out_hi is float [cap_out, Cout] (full fp32 value). */
int b2s_sparse_conv_tc_supported(int cin, int cout);
int b2s_sparse_conv_tc(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride,
                       int rows_in /*row capacity of the feature planes*/, int cin, const b2s_half *w_hi,
                       const b2s_half *w_lo, const int *nbr, int K, const int *num_out_dev, int cap_out,
                       const float *scale, const float *shift, int relu, void *out_hi, b2s_half *out_lo, int out_stride,
                       int cout, unsigned *status_dev, void *stream);

/* Tile plan of a sparse convolution for b2s_sparse_conv_tc_plan (csrc/sparse_plan.cu): the conv kernel owns 128 output
 * rows per CTA and can skip a kernel offset only when NONE of the tile's rows has that neighbour.
 *   tile_mask[t]  bit k: some row of tile t (positions 128t .. 128t+127) has a neighbour through offset k
 *   perm[pos]     (sort = 1) output row at tile position pos: rows are grouped by the shape of their neighbourhood
 *                 (neighbours below / above the centre plane, before / after the centre row; ksize = (kz,ky,kx) names
 *                 the planes) inside chunks of 8192 rows, stable -- roughly halves the (tile, offset) blocks of
 *                 SECOND's middle encoder; sort = 0: tiles in storage order, perm untouched (may be NULL).
 * The convolution result does not depend on the plan (bit-identical with and without). */
int b2s_sparse_tile_plan(const int *nbr, const unsigned *row_mask /*from the rulebook builder, or NULL: read nbr*/, int K,
                         const int *ksize /*[3] or NULL*/, const int *num_out_dev, int cap_out, int sort,
                         int *perm /*[cap_out]*/, unsigned *tile_mask /*[ceil(cap_out/128)]*/, void *stream);
/* b2s_sparse_conv_tc with a tile plan: perm / tile_mask from b2s_sparse_tile_plan (either may be NULL: identity order /
 * every offset). */
int b2s_sparse_conv_tc_plan(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                            const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K, const int *num_out_dev,
                            int cap_out, const int *perm, const unsigned *tile_mask, const float *scale,
                            const float *shift, int relu, void *out_hi, b2s_half *out_lo, int out_stride, int cout,
                            unsigned *status_dev, void *stream);

/* fp32 rows <-> fp16 hi/lo planes (hi = fp16 round-to-nearest, lo = fp16-rounded remainder; saturating).
 * split: x [rows, row_floats] -> out_channels halves per row and plane (>= row_floats, multiple of 8, zero padded), rows
 *        out_stride halves apart (>= out_channels; 2*out_channels for interleaved [row][hi | lo] storage).
 * merge: rows of in_stride halves -> x [rows, row_floats] = hi + lo (exact in fp32).
 * rows = *num_rows_dev (NULL: cap_rows). */
int b2s_split_f16(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows, int row_floats,
                  int out_channels, int out_stride, void *stream);
int b2s_merge_f16(const b2s_half *hi, const b2s_half *lo, float *x, const int *num_rows_dev, int cap_rows,
                  int row_floats, int in_stride, void *stream);

/* ---- dense BEV map ----------------------------------------------------------------------------- */
#define B2S_LAYOUT_NCHW 0 /* out[b, c*D+z, y, x]  (== dense() [B,C,D,H,W] viewed [B,C*D,H,W]) */
#define B2S_LAYOUT_NHWC 1 /* out[b, y, x, c*D+z] */
int b2s_to_bev(const float *feat, const int *coors, const int *num_rows_dev, int cap_rows, int C,
               int batch, int D, int H, int W, float *out, int layout, void *stream);

/* BEV map for the tensor-core RPN: NHWC with a one-pixel zero halo, [B, H+2, W+2, C*D], as two fp16 planes
 * hi = fp16(x), lo = fp16(x - hi) (the 3xF16 split b2s_conv2d_tc consumes).  Rows come as fp32 `feat` [rows, C]
 * (feat_hi/lo NULL) or already split as feat_hi/feat_lo rows of feat_stride halves (feat NULL). */
int b2s_to_bev_tc(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                  const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H, int W,
                  b2s_half *out_hi, b2s_half *out_lo,
                  uint8_t *occupancy /*optional [B,H,W]: 1 where a pixel received data (input of b2s_rpn_bg_plan)*/,
                  void *stream);

/* ---- dense RPN convolution on the tensor pipe (second/pytorch/models/rpn.py:467-497 blocks, :264-299 deblocks,
 *      :386-391 heads): 3x3 stride-1 pad-1 (taps=9) or 1x1 (taps=1) conv + per-channel scale/shift (+ReLU).
 * wgmma implicit GEMM (f16 operands), fp32-grade accuracy through the 3xF16 split (A_lo*B_hi + A_hi*B_lo + A_hi*B_hi,
 * fp32 accumulation in registers, short chains drained with round-to-nearest adds).
 *   in_hi/in_lo  [B, H+2, W+2, Cin]   NHWC + zero halo, fp16 hi/lo planes (Cin multiple of 64)
 *   w_hi/w_lo    [taps, n_pad, Cin]   tap = ky*3+kx, w[tap][co][ci] = W_torch[co][ci][ky][kx] * 2^s (s folded into
 *                                     `scale`); rows >= Cout zero; n_pad in {32, 64, 128}
 *   out_hi       [B, H+2, W+2, out_stride] interior only (out_padded=1) or [B, H, W, out_stride] (out_padded=0);
 *   out_lo       same shape, or NULL: then out_hi is FLOAT and holds the full fp32 value (the heads).
 *   status_dev   may be NULL; B2S_STATUS_F16_RANGE is raised when an output activation exceeds the fp16 range. */
int b2s_conv2d_tc(const b2s_half *in_hi, const b2s_half *in_lo, int batch, int H, int W, int Cin, const b2s_half *w_hi,
                  const b2s_half *w_lo, int taps, int Cout, int n_pad, const float *scale, const float *shift,
                  int relu, void *out_hi, b2s_half *out_lo, int out_padded, int out_stride, unsigned *status_dev,
                  void *stream);

/* general form, for the multi-stage RPNs (rpn.py:469-497: stride-2 first conv of a block after ZeroPad2d(1);
 * :264-299 deblocks: ConvTranspose2d(k = s, stride s) for upsample_stride >= 1, Conv2d(k = s, stride s) below 1;
 * torch.cat of the deblock outputs = channel offsets into one map):
 *   in_hi/in_lo [B, Hin+2, Win+2, Cin] halo-padded.  GEMM pixel (h, w) of the Hg x Wg grid reads input pixels
 *   (h*stride + dy - pad, w*stride + dx - pad), dy < kh, dx < kw (kh*kw <= 16, stride <= 4, pad 0 or 1), weights
 *   [kh*kw, n_pad, Cin], and is written to pixel (h*out_mul + off_h, w*out_mul + off_w) of an Hout x Wout map with
 *   out_stride channels per pixel (pass out pointers already advanced to the first output channel).
 *   ConvTranspose2d k = s: s*s calls with kh = kw = 1, Hg = Hin, out_mul = s, (off_h, off_w) = (a, c), W[:, :, a, c]. */
int b2s_conv2d_tc_ex(const b2s_half *in_hi, const b2s_half *in_lo, int batch, int Hin, int Win, int Cin,
                     const b2s_half *w_hi, const b2s_half *w_lo, int kh, int kw, int stride, int pad, int Cout,
                     int n_pad, const float *scale, const float *shift, int relu, int Hg, int Wg, void *out_hi,
                     b2s_half *out_lo, int Hout, int Wout, int out_padded, int out_stride, int out_mul, int off_h,
                     int off_w,
                     const int *work_list /*optional (device): ids of the 16x16 output tiles to compute, from
                                            b2s_rpn_bg_plan; only for the 3x3 stride-1 128-channel form; NULL: all*/,
                     const int *work_count_dev,
                     const int *bg_list /*optional, with work_list: the background tiles of the output; the kernel's
                                          epilogue warps copy them from the layer's empty-frame response bg_hi/bg_lo
                                          [Hout+2, Wout+2, Cout] while they wait for the tensor pipe (instead of a
                                          separate b2s_rpn_bg_fill launch)*/,
                     const int *bg_count_dev, const b2s_half *bg_hi, const b2s_half *bg_lo, unsigned *status_dev,
                     void *stream);

/* ---- background tiles of the dense RPN ---------------------------------------------------------------
 * The output of layer l of a chain of 3x3 stride-1 pad-1 layers at pixel p depends on the BEV only inside the
 * (2l+1)^2 window around p.  Where that window holds no data the output equals the layer's response to an EMPTY frame
 * at p, a field that depends on the weights only (constant in the interior, different within l pixels of the border).
 * The caller computes that field once per layer by running the layer itself on an empty frame, and keeps it as one
 * halo-padded frame [H+2, W+2, C] of hi/lo planes.
 * b2s_rpn_bg_plan dilates the data mask through `num_layers` consecutive 3x3 stride-1 pad-1 layers and compacts, per
 * layer l, the 16x16 output tiles into
 *   work_lists[l*num_tiles ..]  tiles with a masked pixel (ascending), counts[2l] of them -> b2s_conv2d_tc_ex work_list
 *   bg_lists  [l*num_tiles ..]  background tiles,               counts[2l + 1] of them  -> bg_list / b2s_rpn_bg_fill
 * with num_tiles = batch * ceil(H/16) * ceil(W/16), tile id = (b * tiles_h + th) * tiles_w + tw.
 * scratch: 2*batch*H*W bytes; tile_flags: num_layers*num_tiles ints. */
int b2s_rpn_bg_plan(const uint8_t *occupancy /*[B,H,W]*/, int batch, int H, int W, int num_layers, uint8_t *scratch,
                    int *tile_flags, int *work_lists, int *bg_lists, int *counts, void *stream);
/* copy the listed background tiles of a halo-padded NHWC map [B, H+2, W+2, out_stride] from the layer's empty-frame
 * response f_hi/f_lo [H+2, W+2, C] (fp16 hi/lo planes) */
int b2s_rpn_bg_fill(const int *bg_list, const int *bg_count_dev, int batch, int H, int W, int C, const b2s_half *f_hi,
                    const b2s_half *f_lo, b2s_half *out_hi, b2s_half *out_lo, int out_stride, void *stream);


/* the tail of a single-scale RPNV2 in one kernel (csrc/rpn_tail.cu): y = relu(bn(deblock_1x1(x))) (128 -> 128) never
 * leaves the SM, heads = [box | cls | dir](y) + bias come out as packed fp32 records [B, H, W, out_stride].  Operands as
 * for b2s_conv2d_tc: x = halo-padded fp16 hi/lo planes [B, H+2, W+2, 128]; w1 [128][128], w2 [n_pad2 = 32][128] K-major
 * hi/lo planes, pre-scaled by powers of two folded into scale1 / scale2; shift2 = the heads' bias.  Bit-identical to the
 * two b2s_conv2d_tc launches it replaces (second/pytorch/models/rpn.py:264-299, 386-420). */
int b2s_rpn_tail_tc(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin, const b2s_half *w1_hi,
                    const b2s_half *w1_lo, int Cmid, const float *scale1, const float *shift1, const b2s_half *w2_hi,
                    const b2s_half *w2_lo, int cout2, int n_pad2, const float *scale2, const float *shift2, float *out,
                    int out_stride, unsigned *status_dev, void *stream);

/* ---- PointPillars feature net (single PFNLayer: Linear(F+5 -> Cout, no bias) + BN + ReLU + max) -- */
int b2s_pfn(const float *points, int num_feat, const int *point_slots, const int *num_points_per_voxel,
            const int *coors, const int *num_rows_dev, int cap_rows, int max_points,
            const float *weight /*[Cout, F+5]*/, const float *scale, const float *shift, int cout,
            float vx, float vy, float x_offset, float y_offset, float *out /*[cap_rows,Cout]*/,
            void *stream);

/* ---- box decode + score filter ------------------------------------------------------------------ */
/* Head tensors in the RPN's NCHW conv-output layout: box [B, A_loc*code, H, W], cls [B, A_loc*ncls, H, W],
 * dir [B, A_loc*nbins, H, W] (dir may be NULL).  anchors [A_loc*H*W, code] in (a_loc, y, x) order.
 * anchors_mask [B, A] uint8 may be NULL.  Candidates (score >= thresh) are appended per frame:
 *   cand_box [B,cand_cap,code] decoded, cand_score [B,cand_cap], cand_label/cand_dir [B,cand_cap] int32,
 *   cand_anchor [B,cand_cap] int32 (anchor index, the deterministic tie-break key), cand_count_dev [B]. */
int b2s_decode_filter(const float *box, const float *cls, const float *dir, const float *anchors,
                      const uint8_t *anchors_mask, int batch, int a_loc, int H, int W, int code,
                      int ncls, int nbins, float score_thresh, float *cand_box, float *cand_score,
                      int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev,
                      int cand_cap, unsigned *status_dev, void *stream);

/* same, for head tensors with arbitrary strides (elements): value(b, ch, pixel) = t[b*batch_stride + ch*ch_stride
 * + pixel*pix_stride]; e.g. the packed NHWC record b2s_conv2d_tc writes (box at +0, cls at +14, dir at +16 of a
 * 32-float pixel record: ch_stride 1, pix_stride 32, batch_stride H*W*32 for all three). */
int b2s_decode_filter_strided(const float *box, const float *cls, const float *dir, long long box_batch_stride,
                              long long cls_batch_stride, long long dir_batch_stride, int ch_stride, int pix_stride,
                              const float *anchors, const uint8_t *anchors_mask, int batch, int a_loc, int H, int W,
                              int code, int ncls, int nbins, float score_thresh, float *cand_box,
                              float *cand_score, int *cand_label, int *cand_dir, int *cand_anchor,
                              int *cand_count_dev, int cand_cap, unsigned *status_dev, void *stream);

/* multi-class NMS branch (second/pytorch/models/voxelnet.py:458-547): one candidate list per (class, frame),
 * "virtual frame" v = c*batch + b (class-major): cand_* are [ncls*batch, cand_cap, ...], cand_count_dev [ncls*batch].
 * An anchor joins class c's list when its class-c score passes score_thresh[c] and (class_lo/hi given) its a_loc
 * index lies in [class_lo[c], class_hi[c]) (target_assigner.anchors_range); label = c.  class_lo = class_hi = NULL:
 * nms_class_agnostic.  Head tensors addressed by strides as in b2s_decode_filter_strided.  ncls <= 16.
 * Follow with b2s_nms(batch = ncls*batch) and b2s_concat_class_detections. */
int b2s_decode_filter_multiclass(const float *box, const float *cls, const float *dir, long long box_batch_stride,
                                 long long cls_batch_stride, long long dir_batch_stride, int ch_stride, int pix_stride,
                                 const float *anchors, int batch, int a_loc, int H, int W, int code, int ncls, int nbins,
                                 const int *class_lo /*host[ncls] or NULL*/, const int *class_hi /*host[ncls] or NULL*/,
                                 const float *score_thresh /*host[ncls]*/, float *cand_box, float *cand_score,
                                 int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev, int cand_cap,
                                 unsigned *status_dev, void *stream);
/* det_mc [ncls*batch, post_max, code+2], count_mc [ncls*batch] (class-major b2s_nms outputs) -> per-frame records
 * of up to ncls*post_max rows in class order (voxelnet.py:528-533); det / det_frame_stride / det_count_dev as b2s_nms. */
int b2s_concat_class_detections(const float *det_mc, const int *count_mc, int batch, int ncls, int post_max, int code,
                                float *det, int det_frame_stride, int *det_count_dev, void *stream);

/* ---- top-k + NMS + direction/range epilogue ------------------------------------------------------ */
size_t b2s_nms_workspace_bytes(int batch, int cand_cap, int pre_max);
/* rotated != 0: polygon IoU of BEV boxes (x,y,w,l,r), skip pair when stand-up boxes do not overlap,
 *               suppress when IoU >= iou_thresh;
 * rotated == 0: stand-up boxes of the rotated boxes, IoU with +1 on width/height, suppress when > thresh.
 * Descending score order, ties -> lower anchor index.  Kept boxes (<= post_max per frame), after the
 * direction fix-up and post_center_range test (range_host NULL = no test), are written to
 *   det: frame b's record starts at det + b*det_frame_stride floats and holds post_max rows of
 *        (box[code], score, label); det_frame_stride 0 means post_max*(code+2) (dense [B, post_max, code+2]).
 *        With det_frame_stride > post_max*(code+2) the kept count is ALSO stored as a float in the record's last
 *        element -- the record is then exactly the multi-GPU all-gather payload (SURVEY.md §8e), no packing step;
 *   det_count_dev [B]. */
int b2s_nms(const float *cand_box, const float *cand_score, const int *cand_label, const int *cand_dir,
            const int *cand_anchor, const int *cand_count_dev, int batch, int cand_cap, int code,
            int rotated, int pre_max, int post_max, float iou_thresh, int use_dir, float dir_offset,
            float dir_limit_offset, int num_dir_bins, const float *range_host /*host[6] or NULL*/,
            float *det, int det_frame_stride, int *det_count_dev, void *workspace, size_t workspace_bytes,
            void *stream);

/* numpy-facing spconv.utils signatures: HOST arrays in/out, internal H2D/D2H + sync (like upstream's
 * non_max_suppression, which takes a device_id and does its own copies). */
/* eps=1, inclusive=0: spconv.utils.non_max_suppression ("+1" IoU, suppress if IoU > thresh);
 * eps given, inclusive=1: spconv.utils.non_max_suppression_cpu (suppress if IoU >= thresh). */
/* device_id < 0: run on the caller's current device.  The caller's current device is restored on return. */
int b2s_nms_aligned_host(const float *sorted_dets /*host [N,5]*/, int n, float thresh, float eps,
                         int inclusive, int *keep_out /*host [N]*/, int device_id);
int b2s_nms_rotated_host(const float *corners /*host [N,4,2]*/, const int *order /*host [N]*/,
                         const float *standup_iou /*host [N,N]*/, int n, float thresh,
                         int *keep_out /*host [N]*/, int device_id);


/* ---- rotated overlap matrices (eval / target assignment: SURVEY.md §8(f)2) ------------------------ */
/* criterion -1: IoU, 0: inter/area(box), 1: inter/area(query), 2: intersection area
 * (devRotateIoUEval, second/core/non_max_suppression/nms_gpu.py:553-566). */
/* rotate_iou_gpu_eval replacement (nms_gpu.py:569-607), device resident: boxes [N,5], query_boxes [K,5] as
 * (x, y, w, l, r); out [N,K]; workspace (N+K)*8 floats. */
int b2s_rotate_iou_eval(const float *boxes, int N, const float *query_boxes, int K, int criterion, float *out,
                        float *workspace, void *stream);
/* spconv.utils.rbbox_iou (criterion -1) / rbbox_intersection (criterion 2; interchangeable with
 * rotate_iou_gpu_eval(..., 2) in second/utils/eval.py:174-175) -- HOST arrays: corners [N,4,2], qcorners [K,4,2],
 * standup_iou [N,K]; pairs with standup_iou <= standup_thresh give 0 (second/core/box_np_ops.py:10-34). */
int b2s_rbbox_overlap_host(const float *corners, const float *qcorners, const float *standup_iou, int N, int K,
                           float standup_thresh, int criterion, float *out /*host [N,K]*/, int device_id);

#ifdef __cplusplus
}
#endif
#endif /* B2SECOND_H_ */
