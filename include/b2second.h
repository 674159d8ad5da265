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
 *   b2s_sparse_conv_wgrad, b2s_rulebook_transpose, b2s_from_bev, b2s_split_f16_autoscale
 *                       torch.ops.spconv.indice_conv_backward and the backward of dense() (training:
 *                       second/pytorch/train.py through SubMConv3d / SparseConv3d)
 *   b2s_pfn             PillarFeatureNet.forward (pointpillars.py:203-237, single PFNLayer :51-65)
 *   b2s_pfn_ex          the same, or PillarFeatureNetRadius.forward (pointpillars.py:240-325)
 *   b2s_pfn_train_forward, b2s_pfn_train_backward
 *                       PillarFeatureNet / PillarFeatureNetRadius.forward in train() mode and its autograd backward
 *                       (pointpillars.py:51-65,203-237,290-325): train-mode BatchNorm1d with its running-buffer update
 *   b2s_crop_nhwc       stage0[:, :, c:-c, c:-c] in VoxelNetNuscenesMultiHead.network_forward
 *                       (second/pytorch/models/net_multi_head.py:155-160)
 *   b2s_decode_filter   box_coder.decode_torch + sigmoid + score threshold
 *                       (second/pytorch/models/voxelnet.py:413-414,444,560-576,
 *                        second/pytorch/core/box_torch_ops.py:56-102); _segments: over the torch.cat of several
 *                       heads' predictions (net_multi_head.py:163-172)
 *   b2s_anchor_area_mask
 *                       box_np_ops.sparse_sum_for_anchors_mask + cumsum(0).cumsum(1) +
 *                       box_np_ops.fused_get_anchors_area + `> anchor_area_threshold`
 *                       (second/data/preprocess.py:345-357, second/core/box_np_ops.py:917-946)
 *   b2s_nms             torch.topk + spconv.utils.rotate_non_max_suppression_cpu /
 *                       spconv.utils.non_max_suppression (box_torch_ops.py:454-515,
 *                       second/core/non_max_suppression/nms_cpu.py:20-31, nms_gpu.py:10-19)
 *                       + direction / range epilogue (voxelnet.py:598-628)
 *   b2s_nms_aligned_host, b2s_nms_rotated_host
 *                       the numpy-facing spconv.utils.non_max_suppression /
 *                       rotate_non_max_suppression_cpu signatures (host arrays in, keep list out)
 *   b2s_kitti_convert   KittiDataset.convert_detection_to_kitti_annos (second/data/kitti_dataset.py:37-106)
 *   b2s_kitti_overlaps, b2s_kitti_eval
 *                       calculate_iou_partly + eval_class_v3 behind get_official_eval_result /
 *                       get_coco_eval_result (second/utils/eval.py:362-611,730-916)
 *   b2s_assign_targets  TargetAssigner.assign (second/core/target_assigner.py:38-167) through create_target_np
 *                       (second/core/target_ops.py:29-229), positive_fraction None, for a batch of frames
 *   b2s_augment         the augmentation of prep_pointcloud after database sampling (second/data/preprocess.py:255-294):
 *                       noise_per_object_v3_, random_flip, global_rotation_v2 / scaling_v2 / translate_, the range
 *                       filter, limit_period and the point shuffle (second/core/preprocess.py:153-164,244-273,450-476,
 *                       582-678,749-800,803-899), for a batch of frames
 *   b2s_augment_draws   the random numbers of that augmentation (noise_per_object_v3_'s noises, random_flip,
 *                       global_rotation_v2 / scaling_v2 / translate_ and np.random.shuffle(points)), from a seeded
 *                       Philox stream keyed by (seed, step) and counted by frame instead of numpy's global stream
 *   b2s_db_sample       ground-truth database sampling of prep_pointcloud (second/data/preprocess.py:210-249):
 *                       DataBaseSamplerV2.sample_all / sample_class_v2 collision rejection (second/core/sample_ops.py:
 *                       95-285), points_in_rbbox point removal and the concatenation, for a batch of frames
 *   b2s_detection_loss, b2s_detection_loss_backward
 *                       VoxelNet.loss (second/pytorch/models/voxelnet.py:239-312, second/pytorch/core/losses.py:
 *                       135-294) and the autograd backward of its four differentiable scalars
 *   b2s_optim_step      everything after loss.backward() in the training step (second/pytorch/train.py:299,323-325):
 *                       lr_scheduler.step (torchplus/train/learning_schedules_fastai.py:43-56),
 *                       torch.nn.utils.clip_grad_norm_, OptimWrapper.step (torchplus/train/fastai_optim.py:154-167) over
 *                       torch.optim.Adam (second/pytorch/builder/optimizer_builder.py:68-87) and zero_grad
 *   b2s_train_metrics   VoxelNet.update_metrics (second/pytorch/models/voxelnet.py:654-679, torchplus/metrics.py) and the
 *                       log figures of train.py:335-373; b2s_train_metrics_count / _finish split it so the counts of
 *                       several data-parallel ranks can be added in between (train.py:203-204 multi_gpu)
 *   b2s_pack_sparse_weights
 *                       the tensor-core weight planes of a sparse conv in training (tc.pack_sparse_weights, pow2_scale,
 *                       split_f16 in SparseConvolution._tc_weights / _dgrad_weights) on the device
 *   b2s_split_halo_f16_autoscale, b2s_pack_conv2d_weights, b2s_conv2d_wgrad_tc
 *                       forward and backward of the RPN's 3x3 stride-1 nn.Conv2d layers in training (rpn.py:486-495;
 *                       cuDNN's convolution and its two backward convolutions), with b2s_conv2d_tc_ex
 *   b2s_bn_relu_train_forward, b2s_bn_relu_train_backward
 *                       a train-mode BatchNorm1d / BatchNorm2d followed by ReLU in a Sequential (the RPN's blocks and
 *                       deblocks, rpn.py; the middle encoder's SparseSequential, middle.py:146-191) and their autograd
 *                       backward
 */
#ifndef B2SECOND_H_
#define B2SECOND_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_VERSION 216

/* status bits raised in *status_dev */
#define B2S_STATUS_VOXEL_OVERFLOW 1u   /* more voxels than max_voxels (extra voxels dropped, as spconv) */
#define B2S_STATUS_ROWS_OVERFLOW 2u    /* strided conv produced more rows than cap_out (rows dropped)   */
#define B2S_STATUS_HASH_FULL 4u        /* hash table too small                                            */
#define B2S_STATUS_CAND_OVERFLOW 8u    /* more score-threshold survivors than cand_cap (lowest dropped)  */
#define B2S_STATUS_F16_RANGE 16u       /* an activation left the fp16 range (|x| > 65504) on the tensor-core path;
                                          it was clamped -- results are not fp32-grade for that frame batch      */
#define B2S_STATUS_BAD_INPUT 32u       /* b2s_assign_targets: a frame's gt_offsets are decreasing or past num_gt; that
                                          frame was assigned as if it had no ground truth.  b2s_augment: the same for
                                          gt_offsets or point_offsets, or a perm entry outside its frame.
                                          b2s_db_sample: bad or overlapping point, box or candidate offsets (that
                                          part of the frame is treated as empty), a candidate object id outside the
                                          database or point offsets that disagree with it.  b2s_detection_loss: a
                                          label outside [-1, num_class] (that anchor counts as not cared).
                                          b2s_optim_step: the step counter is outside the hyper-parameter table (the
                                          nearest row was used) or a chunk row is malformed (skipped).
                                          b2s_train_metrics: a label outside [-1, num_class]                      */
#define B2S_STATUS_AUG_BOX_CAP 64u     /* b2s_augment: a frame holds more than B2S_AUGMENT_MAX_BOXES ground truths; its
                                          boxes and points got no per-object noise                               */
#define B2S_STATUS_DB_BOX_CAP 128u     /* b2s_db_sample: a frame's ground truths plus candidates exceed
                                          B2S_DBSAMPLE_MAX_BOXES; that frame got no samples                      */
#define B2S_STATUS_OPT_NONFINITE 256u  /* b2s_optim_step: the gradient norm was inf or NaN; the step was applied as
                                          torch applies it (parameters become NaN)                               */

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
                      const int *padding, const int *dilation, int *coors_out /*[cap_out,4]*/,
                      int *num_out_dev, int cap_out, int *nbr /*[cap_out,K]*/,
                      unsigned long long *hash_keys_out, int *hash_vals_out, int hash_cap_out,
                      void *workspace, size_t workspace_bytes, unsigned *row_mask /*[cap_out] or NULL*/,
                      unsigned *status_dev, void *stream);

/* SubM rulebook of the level b2s_rulebook_conv has JUST produced, read off the occupancy structure that call left in
 * `workspace` (same batch / shape, nothing else run on the workspace in between): coordinate -> row is a bit test +
 * popcount rank, no hash table.  Pass hash_keys_out = hash_vals_out = NULL to b2s_rulebook_conv when every SubM of
 * the produced level is built this way.  nbr as b2s_rulebook_subm, but only its live rows are written (each whole,
 * no prefill of the rest).  At most 27 kernel offsets. */
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

/* same contraction on the tensor pipe (wgmma f16, 3xF16 hi/lo split; accuracy as for b2s_conv2d_tc): Cin in
 * {8,16,32,64}, Cout in {16,32,64}, K <= 27 (b2s_sparse_conv_tc_supported).  Every fp32 operand x travels as two fp16
 * planes hi = fp16(x), lo = fp16(x - hi); per K step the kernel issues A_hi*W_hi + A_hi*W_lo + A_lo*W_hi with fp32
 * accumulation.
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
/* Half-precision mode (the `products` argument of the *_ex entry points below): products = 3 is the 3xF16 form of the
 * entry point without it (hi/lo planes, three wgmma products per K step); products = 1 is the f16 mode: every operand
 * is ONE fp16 plane (hi = fp16 round-to-nearest, saturating), every lo pointer must be NULL, and each K step is one
 * f16 wgmma with fp32 accumulation.  b2s_sparse_conv_tc_plan_ex with products = 1 writes one fp16 plane in out_hi. */
int b2s_sparse_conv_tc_plan_ex(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                               const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K, const int *num_out_dev,
                               int cap_out, const int *perm, const unsigned *tile_mask, const float *scale,
                               const float *shift, int relu, void *out_hi, b2s_half *out_lo, int out_stride, int cout,
                               int products, unsigned *status_dev, void *stream);
/* the same with out_fp32: with products = 1 and out_fp32 = 1 the output is fp32 rows [cap_out, cout] in out_hi (the
 * training forward and input gradient of the f16 mode); out_fp32 must be 0 with products = 3 (out_lo NULL says it). */
int b2s_sparse_conv_tc_plan_ex2(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                                const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K, const int *num_out_dev,
                                int cap_out, const int *perm, const unsigned *tile_mask, const float *scale,
                                const float *shift, int relu, void *out_hi, b2s_half *out_lo, int out_stride, int cout,
                                int products, int out_fp32, unsigned *status_dev, void *stream);

/* fp32 rows <-> fp16 hi/lo planes (hi = fp16 round-to-nearest, lo = fp16-rounded remainder; saturating).
 * split: x [rows, row_floats] -> out_channels halves per row and plane (>= row_floats, multiple of 8, zero padded), rows
 *        out_stride halves apart (>= out_channels; 2*out_channels for interleaved [row][hi | lo] storage).
 * merge: rows of in_stride halves -> x [rows, row_floats] = hi + lo (exact in fp32).
 * rows = *num_rows_dev (NULL: cap_rows). */
int b2s_split_f16(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows, int row_floats,
                  int out_channels, int out_stride, void *stream);
int b2s_merge_f16(const b2s_half *hi, const b2s_half *lo, float *x, const int *num_rows_dev, int cap_rows,
                  int row_floats, int in_stride, void *stream);
/* b2s_split_f16 with products 3 (the same) or 1 (the f16 mode: lo NULL, only hi written) */
int b2s_split_f16_ex(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows, int row_floats,
                     int out_channels, int out_stride, int products, void *stream);
/* b2s_split_f16 of x * 2^e with 2^e chosen on the device from max|x| over the live rows (the b2second.tc.pow2_scale
 * rule: max|x| over the finite elements, max|x| * 2^e in (2^12, 2^13], e clamped to [-126, 126]; 2^e = 1 when no
 * finite element is non-zero) -- for gradients, which are often far below the fp16 normal range.  Unlike b2s_split_f16
 * nothing saturates: +-inf and NaN go through as hi = x, lo = +0, so they reach the result as in fp32 arithmetic.
 * scale_dev [2] floats: [0] <- 2^-e (multiply the tensor-core result by it), [1] is workspace.  Two launches, no host
 * sync. */
int b2s_split_f16_autoscale(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows,
                            int row_floats, int out_channels, int out_stride, float *scale_dev, void *stream);
/* b2s_split_f16_autoscale with products 3 (the same) or 1 (the f16 mode: lo NULL, only hi written, bit-equal to the hi
 * plane of products = 3; the same scale) */
int b2s_split_f16_autoscale_ex(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows,
                               int row_floats, int out_channels, int out_stride, float *scale_dev, int products,
                               void *stream);

/* ---- sparse convolution backward (training) ------------------------------------------------------ */
/* Input gradient (dgrad) is the forward contraction on a transposed table, computed by b2s_sparse_conv /
 * b2s_sparse_conv_tc(_plan) with weights W'[k] = W[k]^T ([K, Cout, Cin]):
 *   SubM (odd kernel): nbr is its own transpose under k <-> K-1-k, so use the same nbr and W'[k] = W[K-1-k]^T;
 *   strided:           use nbrT from b2s_rulebook_transpose and W'[k] = W[k]^T. */
/* nbrT[i][k] = o for nbr[o][k] = i, else -1: the input-side table of a strided conv (for one kernel offset an input row
 * reaches at most one output row).  nbrT [cap_in, K] is filled with -1 first; entries naming a row >= cap_in are
 * dropped and raise B2S_STATUS_ROWS_OVERFLOW (status_dev may be NULL). */
int b2s_rulebook_transpose(const int *nbr, const int *num_out_dev, int cap_out, int K, int *nbrT, int cap_in,
                           unsigned *status_dev, void *stream);
/* Weight gradient dW[k] = sum_o in[nbr[o,k],:]^T dout[o,:] (fp32 FMA, any widths): dW [K, Cin, Cout] (the reference's
 * weight layout viewed flat), times *scale_dev when scale_dev is not NULL (e.g. the 2^-e of a scaled dout).
 * Deterministic (no float atomics): launch 1 writes one partial per 2048-row slab of output rows (rows ascending inside
 * the slab) into the workspace, launch 2 adds the slabs in order. */
size_t b2s_sparse_conv_wgrad_workspace_bytes(int cap_out, int K, int cin, int cout);
int b2s_sparse_conv_wgrad(const float *feat_in, int cin, const float *dout, int cout, const int *nbr, int K,
                          const int *num_out_dev, int cap_out, const float *scale_dev, float *dweight, void *workspace,
                          size_t workspace_bytes, void *stream);
/* the same contraction on the tensor pipe (wgmma f16, 3xF16 split: X_hi*dY_hi + X_hi*dY_lo + X_lo*dY_hi, fp32
 * accumulation): Cin in {8, 16, 32, 64}, Cout in {16, 32, 64}, K <= 27 (the b2s_sparse_conv_tc_supported table).
 *   feat_hi/lo   input rows as for b2s_sparse_conv_tc (in_stride halves, 16-byte aligned);
 *   dout_hi/lo   dY rows (dout_stride halves), e.g. from b2s_split_f16_autoscale with its 2^-e passed as scale_dev;
 *   perm / tile_mask  the forward's tile plan (b2s_sparse_tile_plan; either may be NULL): rows are reduced in perm order,
 *                and 64-row chunks whose tile has none of a K block's offsets are skipped -- bit-identical with and
 *                without tile_mask (same perm);
 *   dweight      [K, Cin, Cout] fp32 (times *scale_dev when not NULL).  Deterministic: fixed chunk chains inside
 *                2048-row slabs, slab partials (workspace) added in order by a second launch. */
size_t b2s_sparse_conv_wgrad_tc_workspace_bytes(int cap_out, int K, int cin, int cout);
int b2s_sparse_conv_wgrad_tc(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                             const b2s_half *dout_hi, const b2s_half *dout_lo, int dout_stride, int cout, const int *nbr,
                             int K, const int *num_out_dev, int cap_out, const int *perm, const unsigned *tile_mask,
                             const float *scale_dev, float *dweight, void *workspace, size_t workspace_bytes,
                             void *stream);
/* b2s_sparse_conv_wgrad_tc with products 3 (the same) or 1 (the f16 mode: feat_lo and dout_lo NULL, one X_hi^T * dY_hi
 * product per k16 step; staging moves half the bytes).  The workspace (b2s_sparse_conv_wgrad_tc_workspace_bytes), the
 * tile_mask skipping and the fixed-order slab sums are those of products = 3. */
int b2s_sparse_conv_wgrad_tc_ex(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                                const b2s_half *dout_hi, const b2s_half *dout_lo, int dout_stride, int cout,
                                const int *nbr, int K, const int *num_out_dev, int cap_out, const int *perm,
                                const unsigned *tile_mask, const float *scale_dev, float *dweight, void *workspace,
                                size_t workspace_bytes, int products, void *stream);

/* ---- dense BEV map ----------------------------------------------------------------------------- */
#define B2S_LAYOUT_NCHW 0 /* out[b, c*D+z, y, x]  (== dense() [B,C,D,H,W] viewed [B,C*D,H,W]) */
#define B2S_LAYOUT_NHWC 1 /* out[b, y, x, c*D+z] */
int b2s_to_bev(const float *feat, const int *coors, const int *num_rows_dev, int cap_rows, int C,
               int batch, int D, int H, int W, float *out, int layout, void *stream);
/* backward of b2s_to_bev: drows[r][c] = dmap at the position b2s_to_bev writes row r, channel c to (same layouts;
 * 0 for rows whose coordinate lies outside the map) */
int b2s_from_bev(const float *dmap, const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D,
                 int H, int W, int layout, float *drows, void *stream);

/* BEV map for the tensor-core RPN: NHWC with a one-pixel zero halo, [B, H+2, W+2, C*D], as two fp16 planes
 * hi = fp16(x), lo = fp16(x - hi) (the 3xF16 split b2s_conv2d_tc consumes).  Rows come as fp32 `feat` [rows, C]
 * (feat_hi/lo NULL) or already split as feat_hi/feat_lo rows of feat_stride halves (feat NULL). */
int b2s_to_bev_tc(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                  const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H, int W,
                  b2s_half *out_hi, b2s_half *out_lo,
                  uint8_t *occupancy /*optional [B,H,W]: 1 where a pixel received data (input of b2s_rpn_block_plan)*/,
                  void *stream);

/* the same scatter into planes kept between calls.  Precondition: the planes are zero except at the pixels flagged in
 * `occupancy` (required), as after zero allocation.  The call zeroes those pixels and clears their flags, then scatters
 * the rows and flags their pixels, so the planes end as b2s_to_bev_tc leaves them and the precondition holds for the
 * next call.  Cost follows the flagged pixels, not the map.  C*D a multiple of 8, planes 16-byte aligned. */
int b2s_to_bev_tc_ex(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                     const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H, int W,
                     b2s_half *out_hi, b2s_half *out_lo, uint8_t *occupancy, void *stream);
/* b2s_to_bev_tc_ex with products 3 (the same) or 1 (the f16 mode: feat_lo and out_lo NULL, one fp16 plane) */
int b2s_to_bev_tc_ex2(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                      const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H, int W,
                      b2s_half *out_hi, b2s_half *out_lo, uint8_t *occupancy, int products, void *stream);

/* ---- dense RPN convolution on the tensor pipe (second/pytorch/models/rpn.py:467-497 blocks, :264-299 deblocks,
 *      :386-391 heads): 3x3 stride-1 pad-1 (taps=9) or 1x1 (taps=1) conv + per-channel scale/shift (+ReLU).
 * wgmma implicit GEMM (f16 operands) with the 3xF16 split (A_lo*B_hi + A_hi*B_lo + A_hi*B_hi, fp32 accumulation in
 * registers, short chains drained with round-to-nearest adds).  Accuracy contract (this kernel and b2s_sparse_conv_tc),
 * per output element y of s * sum(a * w) + shift, with w pre-scaled by the power of two ws, against the exact value y*:
 *     |y - y*| <= |s| * (8 * 2^-23 * S1 + 2^-25 * (Sw + Sa / ws)) + 2^-22 * |y*| + 2^-25,
 *     S1 = sum|a * w|, Sa = sum|a|, Sw = sum|w| over the terms that feed y (before a ReLU, which only shrinks it).
 * That is fp32-grade relative to S1 while |a| >= 2^-3 (and |w| * ws >= 2^-3): below, the fp16 lo plane is subnormal
 * and an operand is good to 2^-25 absolute only (tests/test_gpu_tc_fp64.py pins the bound, tests/tc_ref.py states it).
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
                     const int *work_list /*optional (device): ids of the 8x8 output blocks to compute, from
                                            b2s_rpn_block_plan; only for the 3x3 stride-1 128-channel form; NULL: all*/,
                     const int *work_count_dev,
                     const int *bg_list /*optional, with work_list: the background blocks of the output; the kernel's
                                          fill warps copy them from the layer's empty-frame response bg_hi/bg_lo
                                          [Hout+2, Wout+2, Cout] while its other warps compute the listed blocks*/,
                     const int *bg_count_dev, const b2s_half *bg_hi, const b2s_half *bg_lo, unsigned *status_dev,
                     void *stream);
/* the same with strip lists: work_list / bg_list name output strips 8 pixels wide and list_rows high, list_rows 8
 * (8x8 blocks, b2s_rpn_block_plan; what b2s_conv2d_tc_ex passes), 4 or 2 (b2s_rpn_strip_plan with rows = list_rows).
 * Without a work list list_rows is ignored.  The results are the same bits for either strip height.
 * bg_margin >= 0 promises that the field bg_hi/bg_lo equals its value at pixel (bg_margin, bg_margin) wherever it is at
 * least bg_margin pixels from every border; background strips there are then stored from that value without reading
 * the field.  < 0: every background strip is copied from the field. */
int b2s_conv2d_tc_ex2(const b2s_half *in_hi, const b2s_half *in_lo, int batch, int Hin, int Win, int Cin,
                      const b2s_half *w_hi, const b2s_half *w_lo, int kh, int kw, int stride, int pad, int Cout,
                      int n_pad, const float *scale, const float *shift, int relu, int Hg, int Wg, void *out_hi,
                      b2s_half *out_lo, int Hout, int Wout, int out_padded, int out_stride, int out_mul, int off_h,
                      int off_w, const int *work_list, const int *work_count_dev, const int *bg_list,
                      const int *bg_count_dev, const b2s_half *bg_hi, const b2s_half *bg_lo, int bg_margin,
                      int list_rows, unsigned *status_dev, void *stream);
/* b2s_conv2d_tc_ex2 with products 3 (the same; out_fp32 must be 0, out_lo == NULL selects the fp32 output) or 1 (the
 * f16 mode: in_lo, w_lo, out_lo and bg_lo NULL; the output is one fp16 plane in out_hi, or with out_fp32 = 1 the fp32
 * result, as for the packed heads) */
int b2s_conv2d_tc_ex3(const b2s_half *in_hi, const b2s_half *in_lo, int batch, int Hin, int Win, int Cin,
                      const b2s_half *w_hi, const b2s_half *w_lo, int kh, int kw, int stride, int pad, int Cout,
                      int n_pad, const float *scale, const float *shift, int relu, int Hg, int Wg, void *out_hi,
                      b2s_half *out_lo, int Hout, int Wout, int out_padded, int out_stride, int out_mul, int off_h,
                      int off_w, const int *work_list, const int *work_count_dev, const int *bg_list,
                      const int *bg_count_dev, const b2s_half *bg_hi, const b2s_half *bg_lo, int bg_margin,
                      int list_rows, int products, int out_fp32, unsigned *status_dev, void *stream);

/* ---- background tiles of the dense RPN ---------------------------------------------------------------
 * The output of layer l of a chain of 3x3 stride-1 pad-1 layers at pixel p depends on the BEV only inside the
 * (2l+1)^2 window around p.  Where that window holds no data the output equals the layer's response to an EMPTY frame
 * at p, a field that depends on the weights only (constant in the interior, different within l pixels of the border).
 * The caller computes that field once per layer by running the layer itself on an empty frame, and keeps it as one
 * halo-padded frame [H+2, W+2, C] of hi/lo planes.
 * b2s_rpn_block_plan dilates the data mask through `num_layers` consecutive 3x3 stride-1 pad-1 layers and compacts,
 * per layer l, the 8x8 output blocks into
 *   work_lists[l*num_blocks ..]  blocks with a masked pixel (ascending), counts[2l] of them -> work_list
 *   bg_lists  [l*num_blocks ..]  background blocks,               counts[2l + 1] of them  -> bg_list
 * of b2s_conv2d_tc_ex, with num_blocks = batch * ceil(H/8) * ceil(W/8), block id = (b * blocks_h + bh) * blocks_w + bw.
 * scratch: 2*batch*H*W bytes; block_flags: num_layers*num_blocks ints (1 = the block is computed).
 * b2s_rpn_strip_plan is the same plan over strips 8 pixels wide and `rows` (1, 2, 4 or 8) high: num_strips = batch *
 * ceil(H/rows) * ceil(W/8), strip id = (b * strips_h + sh) * strips_w + sw; rows = 8 gives b2s_rpn_block_plan, and
 * the lists of rows = 4 or 2 go to b2s_conv2d_tc_ex2 with list_rows = rows.
 * b2s_rpn_bg_plan is the same plan over 16x16 tiles (tile_flags / lists of num_tiles = batch * ceil(H/16) * ceil(W/16)
 * entries, tile id = (b * tiles_h + th) * tiles_w + tw); its lists are not accepted by b2s_conv2d_tc_ex. */
int b2s_rpn_block_plan(const uint8_t *occupancy /*[B,H,W]*/, int batch, int H, int W, int num_layers, uint8_t *scratch,
                       int *block_flags, int *work_lists, int *bg_lists, int *counts, void *stream);
int b2s_rpn_strip_plan(const uint8_t *occupancy /*[B,H,W]*/, int batch, int H, int W, int num_layers, int rows,
                       uint8_t *scratch, int *strip_flags, int *work_lists, int *bg_lists, int *counts, void *stream);
int b2s_rpn_bg_plan(const uint8_t *occupancy /*[B,H,W]*/, int batch, int H, int W, int num_layers, uint8_t *scratch,
                    int *tile_flags, int *work_lists, int *bg_lists, int *counts, void *stream);
/* the background strips that must hold the empty-frame response, from the strip_flags of b2s_rpn_strip_plan (same
 * batch, H, W, num_layers, rows), for a chain of layers that ends in the fused tail (b2s_rpn_tail_tc_ex).  Layer l + 1
 * reads layer l only inside the windows of the strips it computes, which reach one pixel into each of the eight
 * neighbouring strips; the tail reads the last layer in tiles of 8 rows x 16 columns (tiles_h = ceil(H/8),
 * tiles_w = ceil(W/16), tile id = (b * tiles_h + th) * tiles_w + tw), and computes a tile iff the last layer computes
 * one of its strips.  Per layer l, band_lists[l*num_strips ..] holds (ascending) the strips layer l does not compute
 * that  - l < num_layers - 1: have a strip computed by layer l + 1 in their 3x3 strip neighbourhood of the same frame,
 *         the strip itself included;
 *       - l = num_layers - 1: lie in a computed tail tile;
 * band_counts[l] of them.  tail_work / tail_bg [num_tiles] get the computed / other tail tiles (ascending),
 * tail_counts[0] / [1] of them.  Passed as bg_list to b2s_conv2d_tc_ex2 and as the lists of b2s_rpn_tail_tc_ex, they
 * leave every pixel a later launch reads, and every head record, as a full fill and a dense tail would. */
int b2s_rpn_strip_bands(const int *strip_flags, int batch, int H, int W, int num_layers, int rows, int *band_lists,
                        int *band_counts, int *tail_work, int *tail_bg, int *tail_counts, void *stream);


/* the tail of a single-scale RPNV2 in one kernel (csrc/rpn_tail.cu): y = relu(bn(deblock_1x1(x))) (128 -> 128) never
 * leaves the SM, heads = [box | cls | dir](y) + bias come out as packed fp32 records [B, H, W, out_stride].  Operands as
 * for b2s_conv2d_tc: x = halo-padded fp16 hi/lo planes [B, H+2, W+2, 128]; w1 [128][128], w2 [n_pad2 = 32][128] K-major
 * hi/lo planes, pre-scaled by powers of two folded into scale1 / scale2; shift2 = the heads' bias.  Bit-identical to the
 * two b2s_conv2d_tc launches it replaces (second/pytorch/models/rpn.py:264-299, 386-420). */
int b2s_rpn_tail_tc(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin, const b2s_half *w1_hi,
                    const b2s_half *w1_lo, int Cmid, const float *scale1, const float *shift1, const b2s_half *w2_hi,
                    const b2s_half *w2_lo, int cout2, int n_pad2, const float *scale2, const float *shift2, float *out,
                    int out_stride, unsigned *status_dev, void *stream);
/* the same with tile lists (from b2s_rpn_strip_bands): only the tiles work_list[0 .. *work_count) are computed, and
 * the records of the tiles bg_list[0 .. *bg_count) are written from `field` [H, W, out_stride], the records the tail
 * gives for an empty frame (this kernel run on the last layer's empty-frame response).  margin >= 0 promises that
 * field equals its record at pixel (margin, margin) wherever it is at least margin pixels from every border.  Other
 * tiles are not written.  NULL lists: every tile is computed (b2s_rpn_tail_tc). */
int b2s_rpn_tail_tc_ex(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin, const b2s_half *w1_hi,
                       const b2s_half *w1_lo, int Cmid, const float *scale1, const float *shift1, const b2s_half *w2_hi,
                       const b2s_half *w2_lo, int cout2, int n_pad2, const float *scale2, const float *shift2,
                       float *out, int out_stride, const int *work_list, const int *work_count, const int *bg_list,
                       const int *bg_count, const float *field, int margin, unsigned *status_dev, void *stream);
/* b2s_rpn_tail_tc_ex with products 3 (the same) or 1 (the f16 mode: in_lo, w1_lo and w2_lo NULL; y is rounded to one
 * fp16 plane before the heads) */
int b2s_rpn_tail_tc_ex2(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin, const b2s_half *w1_hi,
                        const b2s_half *w1_lo, int Cmid, const float *scale1, const float *shift1, const b2s_half *w2_hi,
                        const b2s_half *w2_lo, int cout2, int n_pad2, const float *scale2, const float *shift2,
                        float *out, int out_stride, const int *work_list, const int *work_count, const int *bg_list,
                        const int *bg_count, const float *field, int margin, int products, unsigned *status_dev,
                        void *stream);

/* ---- PointPillars feature net (single PFNLayer: Linear(F+5 -> Cout, no bias) + BN + ReLU + max) -- */
int b2s_pfn(const float *points, int num_feat, const int *point_slots, const int *num_points_per_voxel,
            const int *coors, const int *num_rows_dev, int cap_rows, int max_points,
            const float *weight /*[Cout, F+5]*/, const float *scale, const float *shift, int cout,
            float vx, float vy, float x_offset, float y_offset, float *out /*[cap_rows,Cout]*/,
            void *stream);

/* decoration of the PFN input (b2s_pfn_ex): B2S_PFN_PLAIN = PillarFeatureNet, point features [x, y, z, r, ...] and the
 * Linear has F+5 inputs; B2S_PFN_RADIUS = PillarFeatureNetRadius, point features [sqrt(x*x + y*y), z, r, ...] and F+4
 * inputs.  Both append (xyz - mean xyz) and (xy - pillar centre).  b2s_pfn = b2s_pfn_ex(..., B2S_PFN_PLAIN, ...). */
#define B2S_PFN_PLAIN 0
#define B2S_PFN_RADIUS 1
int b2s_pfn_ex(const float *points, int num_feat, const int *point_slots, const int *num_points_per_voxel,
               const int *coors, const int *num_rows_dev, int cap_rows, int max_points,
               const float *weight /*[Cout, F+5] or [Cout, F+4]*/, const float *scale, const float *shift, int cout,
               float vx, float vy, float x_offset, float y_offset, int decoration, float *out /*[cap_rows,Cout]*/,
               void *stream);

/* ---- PointPillars feature net in training (csrc/pfn_train.cu) ----------------------------------------------------
 * One PFNLayer of PillarFeatureNet (B2S_PFN_PLAIN) or PillarFeatureNetRadius (B2S_PFN_RADIUS) in train() mode
 * (pointpillars.py:51-65,203-237,290-325): Linear(D -> 64, no bias), BatchNorm1d over all N * T slots with batch
 * statistics, ReLU, max over the T slots; D = num_feat + 5 (plain) or + 4 (radius).  The padded [N, T, 64] map is never
 * built: the BN statistics come from the float64 mean mu and covariance C of the decorated inputs d (padded slots are
 * zero rows and count in M = N * T), mean_c = w_c . mu, var_c = w_c^T C w_c, and the weight gradient is the closed form
 *   dW_c = gamma_c s_c (G - A mu - B s_c C w_c),  s_c = 1 / sqrt(var_c + eps),
 * with A = sum delta (= dbeta), B = sum delta xhat (= dgamma), G = sum delta d over the argmax slot of each (n, c),
 * delta = dout[n, c] * [out[n, c] > 0].  No input gradient (the voxels are data).  Sums run in one fixed order in
 * float64 (no float atomics: two runs give the same bits); no entry point syncs, so both can be captured.
 *   voxels      [num_rows, max_points, num_feat] fp32 (the training example's `voxels`); only the first
 *               num_points[n] slots of a row are read, the others are taken as the zero rows upstream masks them to;
 *   num_points  [num_rows] int32; a count outside [1, max_points] raises B2S_STATUS_BAD_INPUT (it is clamped);
 *   coors       [num_rows, 4] int32 (b, z, y, x), 16-byte aligned;  max_points <= 254 (the argmax is one byte);
 *   weight      [64, D] fp32;  gamma, beta [64];  cout must be 64;
 *   running_mean, running_var [64] fp32, num_batches_tracked int64 [1]: updated in place as BatchNorm1d does
 *               (rm = momentum * mean + (1 - momentum) * rm, the variance unbiased by M / (M - 1); nbt += 1);
 *   out         [num_rows, 64] fp32;  argmax [num_rows, 64] uint8: the slot of the maximum, 255 = the padded slot;
 *   workspace   b2s_pfn_train_workspace_bytes(num_rows) (host query) bytes, 16-byte aligned; it carries mu, C and the
 *               per-channel statistics from the forward to the backward, so pass the same workspace to both.
 * Forward: three kernels (moments, statistics and running buffers, output); backward: two (partials, reduce). */
size_t b2s_pfn_train_workspace_bytes(int num_rows);
int b2s_pfn_train_forward(const float *voxels, int num_rows, int max_points, int num_feat, const int *num_points,
                          const int *coors, const float *weight, const float *gamma, const float *beta, int cout,
                          float *running_mean, float *running_var, int64_t *num_batches_tracked, float momentum,
                          float eps, float vx, float vy, float x_offset, float y_offset, int decoration, float *out,
                          uint8_t *argmax, void *workspace, size_t workspace_bytes, unsigned *status_dev,
                          void *stream);
/* dweight [64, D], dgamma, dbeta [64] fp32 from the forward's out, argmax and workspace and dout [num_rows, 64] */
int b2s_pfn_train_backward(const float *voxels, int num_rows, int max_points, int num_feat, const int *num_points,
                           const int *coors, const float *weight, const float *gamma, int cout, float vx, float vy,
                           float x_offset, float y_offset, int decoration, const float *out, const uint8_t *argmax,
                           const float *dout, void *workspace, size_t workspace_bytes, float *dweight, float *dgamma,
                           float *dbeta, void *stream);

/* ---- crop of a halo-padded NHWC map ----------------------------------------------------------------
 * src [B, H+2, W+2, C] (fp16 hi/lo planes, one-pixel halo) -> dst [B, H-2*crop+2, W-2*crop+2, C]: the interior window
 * rows [crop, H-crop), columns [crop, W-crop) of src, with dst's halo written as ZERO -- a conv on dst then sees the
 * zero padding torch applies at the crop edge, not the neighbouring pixels of src.  C % 8 == 0, 16-byte aligned planes. */
int b2s_crop_nhwc(const b2s_half *src_hi, const b2s_half *src_lo, int batch, int H, int W, int C, int crop,
                  b2s_half *dst_hi, b2s_half *dst_lo, void *stream);
/* b2s_crop_nhwc with products 3 (the same) or 1 (the f16 mode: src_lo and dst_lo NULL) */
int b2s_crop_nhwc_ex(const b2s_half *src_hi, const b2s_half *src_lo, int batch, int H, int W, int C, int crop,
                     b2s_half *dst_hi, b2s_half *dst_lo, int products, void *stream);

/* ---- anchor-area mask (second/data/preprocess.py:345-357) ---------------------------------------- */
/* mask_out [batch, num_anchors] uint8 = 1 where the anchor's BEV box holds more than `threshold` voxels.
 * coors [cap, 4] (b, z, y, x), 16-byte aligned; the first min(*num_dev, cap) rows count (the voxels that survived the
 * max_voxels cap), each once at (b, y, x) of a per-frame int32 count map [batch, ny, nx] (ny, nx = grid_size y, x).
 * The map becomes its summed-area table (inclusive prefix sums along x, then y) and, for the box (x0, y0, x1, y1) of
 * anchor_boxes [num_anchors, 4] int32 (16-byte aligned), area = S[y1,x1] - S[y1,x0] - S[y0,x1] + S[y0,x0]: the cells
 * (x0, x1] x (y0, y1], as fused_get_anchors_area reads them.  Boxes must satisfy 0 <= x0 <= x1 < nx and
 * 0 <= y0 <= y1 < ny (b2second/anchor_mask.py derives them on the host in float32).  Counts are integers below 2^24,
 * so the result equals the reference's float32 map bit for bit.  count_map_ws: workspace of
 * b2s_anchor_area_mask_workspace_bytes(batch, ny, nx) (host query) bytes.  One memset and four kernels. */
size_t b2s_anchor_area_mask_workspace_bytes(int batch, int ny, int nx);
int b2s_anchor_area_mask(const int *coors, const int *num_dev, int cap, int batch, int ny, int nx,
                         const int *anchor_boxes, int num_anchors, float threshold, void *count_map_ws,
                         size_t workspace_bytes, uint8_t *mask_out, void *stream);

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

/* several head maps feeding ONE candidate list per frame (VoxelNetNuscenesMultiHead: the large head on the concat map,
 * the small head on the cropped stage-0 map; net_multi_head.py:163-172 concatenates their predictions).  Segment s
 * holds the global anchors [anchor_base, anchor_base + a_loc*H*W) in (a_loc, y, x) order; its tensors are addressed as
 * in b2s_decode_filter_strided (dir may be NULL).  anchors [num_anchors, code] and anchors_mask [B, num_anchors] (may
 * be NULL) are indexed by the GLOBAL anchor id, which is also what cand_anchor holds (the NMS tie-break key).
 * Segments must not overlap; anchors no segment covers never become candidates.  One memset + one launch. */
#define B2S_MAX_HEAD_SEGMENTS 4
typedef struct b2s_head_segment {
    const float *box, *cls, *dir;
    long long box_batch_stride, cls_batch_stride, dir_batch_stride;
    int ch_stride, pix_stride;
    int a_loc, H, W;
    int anchor_base;
} b2s_head_segment;
int b2s_decode_filter_segments(const b2s_head_segment *segments /*host[num_segments]*/, int num_segments,
                               const float *anchors, const uint8_t *anchors_mask, int num_anchors, int batch, int code,
                               int ncls, int nbins, float score_thresh, float *cand_box, float *cand_score,
                               int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev, int cand_cap,
                               unsigned *status_dev, void *stream);

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


/* ---- KITTI detection formatting and evaluation (SURVEY.md §8(f)2) ------------------------------- */
/* Annotations are float64 rows of B2S_KITTI_ROW values, packed frame after frame; frame f owns rows
 * [off[f], off[f+1]) of an int32 offsets array [F+1]:
 *   bbox x1 y1 x2 y2 (0-3), location xyz (4-6), dimensions l h w (7-9), rotation_y (10), alpha (11), score (12),
 *   truncated (13), occluded (14), label (15: class index of a converted detection, unused otherwise).
 * Names are int32 codes: the index of the lower-cased name in the evaluation's class vocabulary, -1 for any other name,
 * B2S_KITTI_DONTCARE for exactly "DontCare". */
#define B2S_KITTI_ROW 16
#define B2S_KITTI_DONTCARE (-2)

/* KittiDataset.convert_detection_to_kitti_annos (second/data/kitti_dataset.py:37-106): det rows of det_stride floats
 * (box[code] as x y z w l h r..., score, label -- the engine's det_record layout), frame f owning [det_off[f],
 * det_off[f+1]); calib [F, 3, 4, 4] float64 (R0_rect, Tr_velo_to_cam, P2 as extended 4x4 matrices); image_shape
 * [F, 2] int32 (H, W).  Boxes whose projected bbox lies off the image are dropped; survivors are compacted per frame in
 * detection order into out rows [det_off[f], det_off[f] + out_count_dev[f]) (truncated = occluded = 0). */
int b2s_kitti_convert(const float *det, int det_stride, int code, const int *det_off, int num_frames,
                      const double *calib, const int *image_shape, double *out, int *out_count_dev, void *stream);

/* calculate_iou_partly's per-frame blocks (second/utils/eval.py:362-445): out[ov_off[f] + j*n_gt_f + i] is the overlap of
 * detection j with ground truth i of frame f (ov_off int64 [F+1], the prefix sum of n_dt_f*n_gt_f).
 * metric 0: image_box_overlap (eval.py:92-119), float64; 1: BEV rotate_iou_gpu_eval (eval.py:122-125), float32;
 * 2: 3D box3d_overlap (eval.py:128-178), float32 rotated intersection times the float64 height overlap, stored through
 * float32.  z_axis / z_center: 1 / 1.0 for camera boxes, 2 / 0.5 for lidar boxes. */
int b2s_kitti_overlaps(int metric, const double *gt, const int *gt_off, const double *dt, const int *dt_off,
                       int num_frames, const long long *ov_off, int z_axis, double z_center, double *out,
                       void *stream);

/* eval_class_v3 for one metric (second/utils/eval.py:479-611, with clean_data :33-89, get_thresholds :11-30,
 * compute_statistics_jit :181-300 and fused_compute_statistics :312-359).  A task is one (class, difficulty,
 * min_overlap): task_info int32 [T, 3] = (class vocabulary id, id that counts as "valid 0" for it -- Van for Car,
 * Person_sitting for Pedestrian -- or -3, difficulty 0..2), task_min_overlap float64 [T].  overlaps / ov_off as
 * b2s_kitti_overlaps writes them.  Outputs float64 [T, 41]: precision and orientation after the running max from the
 * right, and the score thresholds (zero past the last).  Frames are reduced in frame order: bit-reproducible.
 * max_dt_per_frame (host) <= 2048.  workspace: b2s_kitti_eval_workspace_bytes(num_frames, num_gt, num_dt, T).
 * gt_limits / dt_limits uint8 [num_gt] / [num_dt], required when there are boxes: bit d (0..2) set when clean_data
 * puts the box outside difficulty d -- ground truth: occluded > (0, 1, 2)[d] or truncated > (0.15, 0.3, 0.5)[d] or y2 - y1 <= (40, 25, 25)[d];
 * detections: |y2 - y1| < (40, 25, 25)[d] -- compared in the annotation's own dtype, as the reference does (so a
 * float32 height is a float32 difference); the rows' float64 copies of those fields are not read. */
size_t b2s_kitti_eval_workspace_bytes(int num_frames, int num_gt, int num_dt, int num_tasks);
int b2s_kitti_eval(int metric, const double *gt, const int *gt_name, const uint8_t *gt_limits, const int *gt_off,
                   int num_gt, const double *dt, const int *dt_name, const uint8_t *dt_limits, const int *dt_off,
                   int num_dt, int num_frames, int max_dt_per_frame,
                   const double *overlaps, const long long *ov_off, const int *task_info,
                   const double *task_min_overlap, int num_tasks, int compute_aos, double *precision,
                   double *orientation, double *thresholds, void *workspace, size_t workspace_bytes, void *stream);

/* ---- training targets (SURVEY.md §8(f)4) ------------------------------------------------------------ */
/* TargetAssigner.assign (second/core/target_assigner.py:38-167) -> create_target_np (second/core/target_ops.py:29-229)
 * with positive_fraction None, for `batch` frames at once.  The anchor side is fixed per anchor set (b2second.targets
 * builds it once):
 *   anchors [A, box_ndim] float32; anchor_sim [A, 4] float32: rbbox2d_to_near_bbox of the anchor for IoU segments,
 *   (x, y, 0, 0) for distance segments; matched_thr / unmatched_thr [A] float32;
 *   seg_info int32 [S, 4] (anchor_begin, anchor_end, kind 0 = NearestIouSimilarity / 1 = DistanceSimilarity without
 *   rotation, 0) and seg_param float64 [S] (distance_norm) -- one segment per class in per-class mode, one over every
 *   anchor in assign_all; blocks int32 [num_blocks, 4] (segment, anchor_begin, anchor_end, 0), at most 256 anchors each,
 *   covering every segment.
 * Ground truth: gt_boxes [num_gt, box_ndim] float32 (gt_double 0) or float64 (1), frame f owning rows
 * [gt_offsets[f], gt_offsets[f+1]) (device int32 [batch+1]); gt_seg [num_gt] the segment of each GT (-1 or >= S: none);
 * gt_class [num_gt] the label it gives; gt_importance [num_gt] float32 or NULL (ones), indexed with the GT's index
 * within its segment (as assign_per_class passes the unmasked array).  anchors_mask uint8 [batch, A] or NULL.
 * Outputs: labels int32 [batch, A], bbox_targets float32 [batch, A, code_size] (code_size = box_ndim, + 1 when
 * coder_flags bit 1 = vec_encode; bit 0 = linear_dim), importance float32 [batch, A]; optional gt_id int32 [batch, A]
 * (the segment-local GT index of each positive, -1 elsewhere) and overlap float32 [batch, A] (its similarity, 0
 * elsewhere).  Per-GT maxima are integer atomics, everything else is written once: results are bit-reproducible.
 * A segment whose anchors are all pruned gives -1 / 0 / 0 (the reference raises there).  Bad offsets raise
 * B2S_STATUS_BAD_INPUT.  workspace: b2s_assign_targets_workspace_bytes(batch, num_gt, S) (host query) bytes. */
size_t b2s_assign_targets_workspace_bytes(int batch, int num_gt, int num_segments);
int b2s_assign_targets(const float *anchors, const float *anchor_sim, const float *matched_thr,
                       const float *unmatched_thr, int num_anchors, int box_ndim, const int *seg_info,
                       const double *seg_param, int num_segments, const int *blocks, int num_blocks,
                       const void *gt_boxes, int gt_double, int num_gt, const int *gt_offsets, int batch,
                       const int *gt_seg, const int *gt_class, const float *gt_importance,
                       const uint8_t *anchors_mask, int code_size, int coder_flags, int *labels,
                       float *bbox_targets, float *importance, int *gt_id, float *overlap, void *workspace,
                       size_t workspace_bytes, unsigned *status_dev, void *stream);

/* ---- training augmentation (second/data/preprocess.py:255-294) ------------------------------------------------ */
/* Per-object noise without per-object global rotation or groups, the flips, global rotation, scaling and translation, the
 * range filter by centre, limit_period(0.5, 2 pi) and the point shuffle, for `batch` frames.  Random draws are inputs
 * (b2second.augment.draw makes them from a numpy RandomState in the reference's order).
 *   points [num_points, num_feat] float32, frame f owning rows [point_offsets[f], point_offsets[f+1]);
 *   gt_boxes [num_gt, box_ndim] float32 (gt_double 0) or float64 (1), box_ndim 7 or 9 (x y z w l h r [vx vy]), frame f
 *   owning rows [gt_offsets[f], gt_offsets[f+1]); gt_valid uint8 [num_gt] (the class mask: valid boxes get noise and
 *   are kept, the others only block other boxes' tries and are dropped); gt_classes int32, gt_importance float32 (or
 *   NULL: ones) [num_gt], carried to the kept boxes;
 *   loc_noise [num_gt, num_try, 3] / rot_noise [num_gt, num_try] float64, read when object_noise = 1 (0: the
 *   reference's early return when every noise setting is zero -- nothing moves);
 *   frame_params [batch, 8] float64: flip_y, flip_x, translate (0/1, the applied flips and whether the translation
 *   happens), rotation angle, scale, tx, ty, tz;
 *   perm [num_points] int32 frame-local source rows (output row point_offsets[f] + m reads row point_offsets[f] +
 *   perm[point_offsets[f] + m]) or NULL; range_host[4] float32: point_cloud_range[[0, 1, 3, 4]].
 * Outputs: points_out [num_points, num_feat]; point_box int32 [num_points] (the input box row that moved each output
 * point, -1: none) or NULL; boxes_out [num_gt, box_ndim] (input dtype), classes_out, importance_out, src_out (input
 * row) [num_gt]: the kept boxes packed frame after frame in input order, zeros (source row -1) past them; gt_offsets_out int32 [batch + 1]; selected
 * int32 [num_gt]: the chosen try of each box, -1 none, -2 the frame is over the cap.  Pose selection runs one CTA per
 * frame with the frame's corners in shared memory: a frame of more than B2S_AUGMENT_MAX_BOXES boxes raises
 * B2S_STATUS_AUG_BOX_CAP and gets no object noise.  Bad offsets raise B2S_STATUS_BAD_INPUT.  One memset and three
 * kernels; deterministic.  workspace: b2s_augment_workspace_bytes(batch, num_gt, box_ndim) (host query) bytes. */
#define B2S_AUGMENT_MAX_BOXES 1024
size_t b2s_augment_workspace_bytes(int batch, int num_gt, int box_ndim);
int b2s_augment(const float *points, int num_points, int num_feat, const int *point_offsets, int batch,
                const void *gt_boxes, int gt_double, int box_ndim, int num_gt, const int *gt_offsets,
                const uint8_t *gt_valid, const int *gt_classes, const float *gt_importance, const double *loc_noise,
                const double *rot_noise, int num_try, int object_noise, const double *frame_params, const int *perm,
                const float *range_host, float *points_out, int *point_box, void *boxes_out, int *gt_offsets_out,
                int *classes_out, float *importance_out, int *src_out, int *selected, void *workspace,
                size_t workspace_bytes, unsigned *status_dev, void *stream);

/* ---- device draws of the training augmentation ------------------------------------------------------------------ */
/* The random numbers b2s_augment reads, drawn on the device instead of from numpy's stream: noise_per_object_v3_'s
 * loc_noises and rot_noises, random_flip's choices, global_rotation_v2's and global_scaling_v2's uniforms and
 * global_translate_'s normals (second/core/preprocess.py:582-678,749-800,885-899), and preprocess.py's
 * np.random.shuffle(points).  Every value is a function of (seed, *step_dev, frame, stream, index):
 *   block function Philox4x64-10 (numpy.random.Philox's), key (seed, step), counter (frame, stream, index, 0) with
 *   frame = frame_base + b for batch-local frame b; u(w) = (w >> 11) 2^-53; a uniform on [lo, hi) is lo + (hi - lo) u;
 *   normals by Box-Muller from words (wa, wb): r = sqrt(-2 ln(1 - u(wa))), t = 2 pi u(wb), the pair (r cos t, r sin t).
 *   loc_noise[g, t] (box b of its frame, try t): block (f, 0, 100 b + t), normals (w0, w1) -> n0, n1 and (w2, w3) ->
 *   n2 (the cos term), times loc_std; rot_noise[g, t]: uniform(rot_noise) from w0 of block (f, 1, 100 b + t).
 *   frame_params[b] (b2s_augment's layout): block (f, 2, 0, 0): flip_x = u(w0) < 0.5, flip_y = u(w1) < 0.5 (each only
 *   where random_flip_x / _y is set), angle = uniform(rotation) from w2, scale = uniform(scaling) from w3; when a
 *   translate_std is nonzero, translate = 1 and block (f, 2, 1, 0)'s normals as loc_noise's times (translate_std[0],
 *   translate_std[1], translate_std[0]) (global_translate_ draws z with std[0]); otherwise translate = 0, t = 0.
 *   perm: the frame-local permutation pi of a frame of n points: k >= 1 the smallest with 4^k >= n, x < 4^k split
 *   into (L, R) = (x >> k, x & (2^k - 1)), 4 rounds (L, R) <- (R, L ^ (w0 of block (f, 3, r, R) & (2^k - 1))) for
 *   r = 0..3, repeated while the result is >= n; perm[point_offsets[b] + i] = pi(i); n <= 1 keeps the identity.
 * Each row finds its frame by searching gt_offsets / point_offsets [batch + 1] (device); rows outside every frame, or
 * in a frame whose range is malformed, get zeros.  loc_noise [num_gt, B2S_AUGMENT_NUM_TRY, 3] and rot_noise [num_gt,
 * B2S_AUGMENT_NUM_TRY] float64 are written when params_host->object_noise (else may be NULL); frame_params [batch, 8]
 * float64; perm int32 [num_points], or NULL: no shuffle.  step_dev: uint64 device counter, read by every kernel of the
 * call and advanced by one at its end, so a captured call draws the next step at every replay.  No host sync, no
 * atomics; deterministic.  Four kernels at most. */
#define B2S_AUGMENT_NUM_TRY 100
typedef struct {
    double loc_std[3];          /* groundtruth_localization_noise_std */
    double rot_noise[2];        /* groundtruth_rotation_uniform_noise */
    double rotation[2];         /* global_rotation_uniform_noise */
    double scaling[2];          /* global_scaling_uniform_noise */
    double translate_std[3];    /* global_translate_noise_std */
    int object_noise;           /* 1: noise_per_object_v3_ draws (b2second.augment.object_noise_enabled) */
    int random_flip_x, random_flip_y;
} b2s_augment_draw_params;
int b2s_augment_draws(uint64_t seed, uint64_t *step_dev, uint64_t frame_base, int batch, const int *gt_offsets,
                      int num_gt, const int *point_offsets, int num_points, const b2s_augment_draw_params *params_host,
                      double *loc_noise, double *rot_noise, double *frame_params, int *perm, void *stream);

/* ---- training ground-truth database sampling (second/data/preprocess.py:210-249) ----------------------------- */
/* The device half of DataBaseSamplerV2.sample_all without group sampling, per-object rotation or random crop, for
 * `batch` frames.  The candidates are inputs (b2second.dbsample.draw makes them from a numpy RandomState in the
 * reference's order); this call decides which are accepted and builds the frames prep_pointcloud holds at
 * preprocess.py:249.
 *   points / point_offsets / gt_boxes / gt_offsets / gt_valid / gt_classes / gt_importance: as b2s_augment's inputs
 *   (gt_importance NULL: ones); every gt row of a frame blocks candidates, whatever its class mask;
 *   cand_obj int32 [num_cand] database object ids, frame f owning rows [cand_offsets[f], cand_offsets[f+1]), class by
 *   class in sample-group order; cand_group int32 [num_cand] the sample group of each (equal values: one class);
 *   cand_point_offsets int32 [num_cand + 1] the prefix of the candidates' point counts (num_cand_points the total);
 *   db_points [*, num_feat] float32, object o owning rows [db_point_offsets[o], db_point_offsets[o+1]) (int64, the
 *   object's points relative to its box centre); db_boxes [num_objects, box_ndim] in the gt dtype; db_classes int32
 *   [num_objects] 1-based class ids (class_names.index(name) + 1); sample_importance, remove_points 0/1
 *   (remove_points_after_sample: a frame point inside an accepted box is dropped).
 * A candidate is rejected when its BEV box collides with a gt box of its frame, an accepted candidate of an earlier
 * class, an accepted earlier candidate of its own class, or any later candidate of its own class (dbsample.cu states
 * why).  Outputs, packed frame after frame: points_out [num_points + num_cand_points, num_feat] (the accepted
 * objects' points translated by their box centre in acceptance order, then the frame's kept points in order; zeros
 * past point_offsets_out[batch]), point_offsets_out int32 [batch + 1]; boxes_out [num_gt + num_cand, box_ndim],
 * valid_out uint8, classes_out int32, importance_out float32, src_object int32 (the database object, -1 for the
 * frame's own rows) [num_gt + num_cand]: the frame's rows then its accepted ones (zeros past gt_offsets_out[batch]),
 * gt_offsets_out int32 [batch + 1] -- b2s_augment's input layout; accepted uint8 [num_cand].  A frame whose gt rows
 * plus candidates exceed B2S_DBSAMPLE_MAX_BOXES raises B2S_STATUS_DB_BOX_CAP and gets no samples.  A frame's range in
 * an offsets array is used only when it is ordered, inside the array, and neither before an earlier entry nor after a
 * later one (so the ranges in use never overlap); otherwise that part of the frame is empty.  Such ranges, object ids
 * outside the database and cand_point_offsets steps that differ from the objects' point counts (those candidates are
 * rejected) raise B2S_STATUS_BAD_INPUT; no output is written past its capacity.  Four memsets and five kernels; no
 * sync, deterministic.  workspace:
 * b2s_db_sample_workspace_bytes(batch, num_points, num_cand) (host query) bytes. */
#define B2S_DBSAMPLE_MAX_BOXES 1024
size_t b2s_db_sample_workspace_bytes(int batch, int num_points, int num_cand);
int b2s_db_sample(const float *points, int num_points, int num_feat, const int *point_offsets, int batch,
                  const void *gt_boxes, int gt_double, int box_ndim, int num_gt, const int *gt_offsets,
                  const uint8_t *gt_valid, const int *gt_classes, const float *gt_importance, const int *cand_obj,
                  const int *cand_group, const int *cand_offsets, const int *cand_point_offsets, int num_cand,
                  int num_cand_points, const float *db_points, const long long *db_point_offsets,
                  const void *db_boxes, const int *db_classes, int num_objects, float sample_importance,
                  int remove_points, float *points_out, int *point_offsets_out, void *boxes_out, int *gt_offsets_out,
                  uint8_t *valid_out, int *classes_out, float *importance_out, int *src_object, uint8_t *accepted,
                  void *workspace, size_t workspace_bytes, unsigned *status_dev, void *stream);

/* ---- training loss (second/pytorch/models/voxelnet.py:239-312) ------------------------------------------------- */
/* VoxelNet.loss with the loss settings of every config: WeightedSmoothL1LocalizationLoss (second/pytorch/core/losses.py:
 * 135-182) on the sin-encoded box (add_sin_difference, voxelnet.py:704-714), SigmoidFocalClassificationLoss
 * (losses.py:184-192,236-294) on the one-hot target without background (voxelnet.py:255,737-741), NormByNumPositives
 * weights times importance (prepare_loss_weights, voxelnet.py:756-795, :265-267), the reductions and _get_pos_neg_loss
 * (voxelnet.py:20-34,275-282), and the softmax direction loss (get_direction_target, voxelnet.py:814-828, :284-297)
 * weighted by positive importance over its per-frame sum.  Settings, read on the host: */
typedef struct b2s_loss_params {
    float alpha, gamma;            /* focal */
    float sigma;                   /* smooth L1 */
    float code_weight[7];
    float pos_cls_weight, neg_cls_weight;
    float loc_weight, cls_weight, dir_weight;   /* localization_weight, classification_weight, direction_loss_weight */
    float sin_factor;              /* sin_error_factor */
    float dir_offset;
    int num_dir_bins;
} b2s_loss_params;
/* Inputs: box_preds [batch, A, 7], cls_preds [batch, A, num_class], dir_preds [batch, A, num_dir_bins] float32 (the
 * heads' permuted outputs, contiguous); labels [batch, A] int32 (labels_int64 0) or int64 (1): -1 ignore, 0 background,
 * c >= 1 class c; reg_targets [batch, A, 7], importance [batch, A], anchors [batch, A, 7] (only the yaw is read).
 * Outputs: reduced float32 [4] = loss, cls_loss_reduced, loc_loss_reduced, dir_loss_reduced (unweighted; loss holds it
 * times dir_weight); pos_neg [2] = cls_pos_loss, cls_neg_loss; optional (NULL: not written) cls_loss [batch, A,
 * num_class], loc_loss [batch, A, 7], cared uint8 [batch, A]; norms [batch, 2] = max(positives, 1) and max(sum of
 * positive importance, 1) per frame, which the backward reads.  A label outside [-1, num_class] counts as -1 and
 * raises B2S_STATUS_BAD_INPUT.  Three kernels; sums in one fixed order (no float atomics), so results are
 * bit-reproducible; no sync.  workspace: b2s_detection_loss_workspace_bytes(batch, A) (host query) bytes. */
size_t b2s_detection_loss_workspace_bytes(int batch, int num_anchors);
int b2s_detection_loss(const float *box_preds, const float *cls_preds, const float *dir_preds, int num_class,
                       int num_dir_bins, const void *labels, int labels_int64, const float *reg_targets,
                       const float *importance, const float *anchors, int batch, int num_anchors,
                       const b2s_loss_params *params, float *reduced, float *pos_neg, float *cls_loss,
                       float *loc_loss, uint8_t *cared, float *norms, void *workspace, size_t workspace_bytes,
                       unsigned *status_dev, void *stream);
/* The gradient of d_reduced[0] * loss + d_reduced[1] * cls_loss_reduced + d_reduced[2] * loc_loss_reduced +
 * d_reduced[3] * dir_loss_reduced (d_reduced: device float32 [4], or NULL for zeros) in the preds, written to d_box,
 * d_cls, d_dir in the preds' layout; the inputs and norms as the forward had them.  One kernel, one thread per anchor;
 * an anchor of weight 0 gets exactly 0. */
int b2s_detection_loss_backward(const float *box_preds, const float *cls_preds, const float *dir_preds, int num_class,
                                int num_dir_bins, const void *labels, int labels_int64, const float *reg_targets,
                                const float *importance, const float *anchors, int batch, int num_anchors,
                                const b2s_loss_params *params, const float *norms, const float *d_reduced,
                                float *d_box, float *d_cls, float *d_dir, void *stream);

/* ---- optimizer step (second/pytorch/train.py:299,323-325) -------------------------------------------------------- */
/* One training step's work after loss.backward(), for all parameter tensors in two kernels: the L2 norm of all
 * gradients and g *= min(1, max_norm / (norm + 1e-6)) (torch.nn.utils.clip_grad_norm_, train.py:323); weight decay,
 * decoupled (fixed_weight_decay: p *= 1 - wd * lr before Adam, torchplus/train/fastai_optim.py:157-166) or L2 inside
 * Adam (g += wd * p); torch.optim.Adam's update with amsgrad off (optimizer_builder.py:68-76, train.py:324); zero_grad
 * (train.py:325); and the schedule's advance (lr_scheduler.step, train.py:299).  All tensors are float32.
 * The hyper-parameters that change per step come from device memory: hyper [settings->total_step,
 * B2S_OPTIM_HYPER_COLS] float64, row s for the step taken when *step_dev == s: lr, beta1, 1 - beta1^(s+1),
 * sqrt(1 - beta2^(s+1)), 1 - wd * lr.  *step_dev (int64) is read by the first kernel and written back + 1 by the
 * second, so a captured call advances the schedule by itself when replayed; past the table the last row is used and
 * B2S_STATUS_BAD_INPUT raised.  Settings, read on the host: */
#define B2S_OPTIM_CHUNK 4096       /* elements of one tensor one CTA handles */
#define B2S_OPTIM_HYPER_COLS 5
typedef struct b2s_optim_params {
    double weight_decay, beta2, eps;
    double max_norm;               /* clip_grad_norm_'s max_norm */
    long long total_step;          /* rows of hyper */
    int decoupled;                 /* 1: fixed_weight_decay (p *= hyper[4]); 0: L2 (g += weight_decay * p) */
    int zero_grad;                 /* 1: write zeros into every gradient after it is used */
} b2s_optim_params;
/* params, grads, exp_avg, exp_avg_sq: device arrays of num_tensors device pointers; a NULL grads entry is a parameter
 * without gradient (decayed in the decoupled form, otherwise untouched, as torch skips it).  chunks: device int32
 * [num_chunks, 4], 16-byte aligned, rows (tensor, first element, elements <= B2S_OPTIM_CHUNK, 0) that tile every
 * tensor once; tensors whose four pointers are 16-byte aligned at a chunk's start move as 16-byte words.  total_norm:
 * device float32 [1], the norm before clipping.  A non-finite norm propagates as in torch (a NaN norm makes every
 * parameter NaN) and raises B2S_STATUS_OPT_NONFINITE.  Sums run in one fixed order (float64 partials per chunk, no float
 * atomics) and every float32 operation is a round-to-nearest intrinsic, so results are bit-reproducible; no sync.
 * workspace: b2s_optim_workspace_bytes(num_chunks) (host query) bytes. */
size_t b2s_optim_workspace_bytes(int num_chunks);
int b2s_optim_step(float *const *params, float *const *grads, float *const *exp_avg, float *const *exp_avg_sq,
                   int num_tensors, const int *chunks, int num_chunks, const double *hyper, long long *step_dev,
                   const b2s_optim_params *settings, float *total_norm, void *workspace, size_t workspace_bytes,
                   unsigned *status_dev, void *stream);

/* ---- training metrics (second/pytorch/models/voxelnet.py:654-679, second/pytorch/train.py:327-373) -------------- */
/* One step of VoxelNet.update_metrics through torchplus/metrics.py (Accuracy, PrecisionRecall, Scalar) with sigmoid
 * scores and background encoded as zeros, plus the log figures train.py:335-373 computes.  Settings, read on the
 * host: */
#define B2S_METRICS_MAX_THRESHOLDS 16
#define B2S_METRICS_MAX_CODE 8
typedef struct b2s_metrics_params {
    int num_thresholds;
    float thresholds[B2S_METRICS_MAX_THRESHOLDS];   /* rpn_metrics.thresholds as float32 (score > threshold) */
    float acc_threshold;                            /* rpn_acc._threshold (0.5) */
} b2s_metrics_params;
/* The reference's running buffers (device float32, updated in place): rpn_acc.total / count [1],
 * rpn_metrics.prec_total / prec_count / rec_total / rec_count [num_thresholds], rpn_cls_loss.total / count and
 * rpn_loc_loss.total / count [1].  Pointers read on the host. */
typedef struct b2s_metrics_buffers {
    float *acc_total, *acc_count;
    float *prec_total, *prec_count, *rec_total, *rec_count;
    float *cls_total, *cls_count, *loc_total, *loc_count;
} b2s_metrics_buffers;
/* record: float32 [B2S_METRICS_RECORD_HEAD + 2 * num_thresholds]; after the head, prec[T] then rec[T] */
#define B2S_METRICS_REC_ACC 0           /* rpn_acc.total / count */
#define B2S_METRICS_REC_CLS 1           /* rpn_cls_loss.total / count */
#define B2S_METRICS_REC_CLS_RT 2        /* *cls_loss */
#define B2S_METRICS_REC_LOC 3           /* rpn_loc_loss.total / count */
#define B2S_METRICS_REC_LOC_RT 4        /* *loc_loss */
#define B2S_METRICS_REC_CLS_POS_RT 5    /* *cls_pos_loss (0 when NULL) */
#define B2S_METRICS_REC_CLS_NEG_RT 6    /* *cls_neg_loss (0 when NULL) */
#define B2S_METRICS_REC_DIR_RT 7        /* *dir_loss (0 when NULL) */
#define B2S_METRICS_REC_NUM_POS 8       /* labels > 0 in frame 0 */
#define B2S_METRICS_REC_NUM_NEG 9       /* labels == 0 in frame 0 */
#define B2S_METRICS_REC_NUM_ANCHORS 10  /* anchors_mask set in frame 0 (num_anchors when NULL) */
#define B2S_METRICS_REC_LOC_ELEM 11     /* [B2S_METRICS_MAX_CODE]: loc_loss_elem[:, :, j] summed / batch (0 past code) */
#define B2S_METRICS_RECORD_HEAD 19
/* Inputs: cls_preds [batch, A, num_class] float32; labels [batch, A] int32 (labels_int64 0) or int64 (1); cared
 * uint8 [batch, A] (the loss's `cared`, the metrics' weights); cls_loss, loc_loss: device float32 scalars
 * (cls_loss_reduced, loc_loss_reduced).  Optional (NULL): loc_loss_elem [batch, A, code_size] (the loss's per-element
 * loc_loss), anchors_mask uint8 [batch, A], and the device scalars cls_pos_loss, cls_neg_loss, dir_loss.  The score is
 * max_c sigmoid(pred_c) with torch's float32 sigmoid; Accuracy counts pred == label over all anchors, unweighted, as
 * Accuracy.forward does.  A label outside [-1, num_class] raises B2S_STATUS_BAD_INPUT (it is counted as the reference
 * counts it).  Two kernels: one pass over cls_preds, labels and cared with per-CTA integer counts, then one CTA that adds
 * them in a fixed order, updates the buffers and writes the record; bit-reproducible, no sync.  Per-step counts must
 * stay below 2^24 (as the reference's float32 sums need).  workspace: b2s_train_metrics_workspace_bytes(batch, A) bytes. */
size_t b2s_train_metrics_workspace_bytes(int batch, int num_anchors);
int b2s_train_metrics(const float *cls_preds, int num_class, const void *labels, int labels_int64, const uint8_t *cared,
                      int batch, int num_anchors, const b2s_metrics_params *params, const float *cls_loss,
                      const float *loc_loss, const float *loc_loss_elem, int code_size, const uint8_t *anchors_mask,
                      const float *cls_pos_loss, const float *cls_neg_loss, const float *dir_loss,
                      const b2s_metrics_buffers *buffers, float *record, void *workspace, size_t workspace_bytes,
                      unsigned *status_dev, void *stream);
/* The same step in two halves, so the counts of several shares of a batch (one per data-parallel rank) can be added
 * before the buffers are updated.  b2s_train_metrics_count takes b2s_train_metrics' inputs and writes this share's
 * count record, float32 [B2S_METRICS_COUNT_HEAD + 2 * num_thresholds]: */
#define B2S_METRICS_CNT_FRAMES 0        /* batch */
#define B2S_METRICS_CNT_CORRECT 1       /* anchors with pred == label (Accuracy's total) */
#define B2S_METRICS_CNT_CARED 2         /* cared anchors */
#define B2S_METRICS_CNT_POS 3           /* cared anchors with label > 0 */
#define B2S_METRICS_CNT_NUM_POS 4       /* labels > 0 in frame 0 (0 when has_frame0 is 0) */
#define B2S_METRICS_CNT_NUM_NEG 5       /* labels == 0 in frame 0 (0 when has_frame0 is 0) */
#define B2S_METRICS_CNT_NUM_ANCHORS 6   /* anchors_mask set in frame 0 (0 when has_frame0 is 0) */
#define B2S_METRICS_CNT_CLS_LOSS 7      /* *cls_loss */
#define B2S_METRICS_CNT_LOC_LOSS 8      /* *loc_loss */
#define B2S_METRICS_CNT_CLS_POS 9       /* *cls_pos_loss (0 when NULL) */
#define B2S_METRICS_CNT_CLS_NEG 10      /* *cls_neg_loss (0 when NULL) */
#define B2S_METRICS_CNT_DIR 11          /* *dir_loss (0 when NULL) */
#define B2S_METRICS_CNT_LOC_ELEM 12     /* [B2S_METRICS_MAX_CODE]: loc_loss_elem[:, :, j] summed (float64, rounded once) */
#define B2S_METRICS_COUNT_HEAD 20       /* then tp[T] and fp[T]: cared positives / negatives scored above each threshold */
/* Every count is an integer below 2^24, so the float32 records of several shares add exactly.  Summed over W shares,
 * the five loss slots hold W times the replica mean, which b2s_train_metrics_finish scales back by loss_scale (1/W).
 * b2s_train_metrics_finish reads such a (possibly summed) record on the device, updates the running buffers in the
 * reference's order and writes the record b2s_train_metrics writes; with loss_scale 1, count followed by finish on one
 * share is b2s_train_metrics bit for bit.  loc_elem of the log record is the summed slot over the summed frame count.
 * No sync; finish needs no workspace. */
int b2s_train_metrics_count(const float *cls_preds, int num_class, const void *labels, int labels_int64,
                            const uint8_t *cared, int batch, int num_anchors, const b2s_metrics_params *params,
                            const float *cls_loss, const float *loc_loss, const float *loc_loss_elem, int code_size,
                            const uint8_t *anchors_mask, const float *cls_pos_loss, const float *cls_neg_loss,
                            const float *dir_loss, int has_frame0, float *counts, void *workspace,
                            size_t workspace_bytes, unsigned *status_dev, void *stream);
int b2s_train_metrics_finish(const float *counts, const b2s_metrics_params *params, float loss_scale,
                             const b2s_metrics_buffers *buffers, float *record, void *stream);

/* ---- sparse conv weights on the tensor pipe (b2second/tc.py: pack_sparse_weights, pow2_scale, split_f16) -------- */
/* w [K, cin, cout] float32 (spconv's layout) -> the fp16 hi/lo planes b2s_sparse_conv_tc(_plan) takes as its B operand,
 * bit-identical to tc.split_f16(tc.pack_sparse_weights(L), tc.pow2_scale(...)) with L[k] = w[k] (transpose 0) or
 * L[k] = w[flip ? K-1-k : k]^T (transpose 1: the input gradient's weights).  With n_in x n_out the channels of L, the
 * planes are [ceil(K / P), n_out, 64] halves, P = 64 / n_in' kernel offsets per 128-byte K block, n_in' = n_in padded to
 * 8 (n_in in 1..8, 16, 32, 64).  scale_dev: device float32 [3]; [0] = s, the power of two with max|w| * s in
 * (2^12, 2^13] over the finite weights, clamped to [2^-126, 2^126] (1 when no finite weight is non-zero), [1] = 1/s,
 * [2] scratch.  A non-finite weight is packed as itself (hi = w, lo = +0; tc.split_f16 would saturate it), so the planes
 * equal the host path's for finite weights.  A memset and two kernels (max|w| as integer atomicMax on the bit patterns,
 * then the pack and split); no sync. */
int b2s_pack_sparse_weights(const float *w, int K, int cin, int cout, int transpose, int flip, b2s_half *hi,
                            b2s_half *lo, float *scale_dev, void *stream);
/* with products 3 (the same) or 1 (the f16 mode: lo NULL, only hi written, bit-equal to the hi plane of products = 3) */
int b2s_pack_sparse_weights_ex(const float *w, int K, int cin, int cout, int transpose, int flip, b2s_half *hi,
                               b2s_half *lo, float *scale_dev, int products, void *stream);

/* ---- dense RPN training: 3x3 stride-1 pad-1 convolutions on the tensor pipe (csrc/conv_train.cu) ------------------
 * Forward y = conv(x, W) and input gradient dX = conv(dY, W') with W'[tap] = W[8 - tap]^T are b2s_conv2d_tc_ex
 * launches (kh = kw = 3, stride 1, pad 1, fp32 output: out_lo NULL) on the planes below; the weight gradient is
 * b2s_conv2d_wgrad_tc.  No entry point syncs, so a training step that uses them can be captured. */
/* fp32 map x, [B, C, H, W] (layout B2S_LAYOUT_NCHW) or [B, H, W, C] (B2S_LAYOUT_NHWC, 16-byte aligned) -> x * 2^e as
 * fp16 hi/lo planes [B, H+2, W+2, C] with a zero halo (the input b2s_conv2d_tc_ex and b2s_conv2d_wgrad_tc read), with e
 * picked on the device from max|x| by the b2s_split_f16_autoscale rule.  C multiple of 8.  scale_dev [2] floats: [0] <-
 * 2^-e, [1] workspace.  A non-finite element goes through as hi = x, lo = +0 (as in b2s_split_f16_autoscale) and raises
 * B2S_STATUS_F16_RANGE (status_dev may be NULL).  A memset, two kernels. */
int b2s_split_halo_f16_autoscale(const float *x, int layout, int batch, int C, int H, int W, b2s_half *hi, b2s_half *lo,
                                 float *scale_dev, unsigned *status_dev, void *stream);
/* with products 3 (the same) or 1 (the f16 mode: lo NULL, only hi written, bit-equal to the hi plane of products = 3) */
int b2s_split_halo_f16_autoscale_ex(const float *x, int layout, int batch, int C, int H, int W, b2s_half *hi,
                                    b2s_half *lo, float *scale_dev, unsigned *status_dev, int products, void *stream);
/* torch weight w [cout, cin, 3, 3] fp32 -> the b2s_conv2d_tc_ex weight planes, scaled by the power of two s with
 * max|w| * s in (2^12, 2^13] (as b2s_pack_sparse_weights, non-finite weights and the clamp included; scale_dev [3]:
 * [0] = s, [1] = 1/s, [2] scratch).
 * transpose 0: L[tap][o][i] = w[o][i][tap] (n_out = cout, n_in = cin, the forward); transpose 1: L[tap][o][i] =
 * w[i][o][8 - tap] (n_out = cin, n_in = cout, the input gradient).  Planes [G][9][n_pad][n_in] halves with G =
 * ceil(n_out / 128) launches of up to 128 output channels, n_pad = min(n_out, 128), zero rows past n_out.  cin, cout
 * multiples of 64.  The epilogue scale of a launch is (the input planes' 2^-e) * (1/s). */
int b2s_pack_conv2d_weights(const float *w, int cout, int cin, int transpose, b2s_half *hi, b2s_half *lo,
                            float *scale_dev, void *stream);
/* with products 3 (the same) or 1 (the f16 mode: lo NULL, only hi written, bit-equal to the hi plane of products = 3) */
int b2s_pack_conv2d_weights_ex(const float *w, int cout, int cin, int transpose, b2s_half *hi, b2s_half *lo,
                               float *scale_dev, int products, void *stream);
/* dW[co][ci][ky][kx] = sum_px dY[px][co] * X[px + (ky - 1, kx - 1)][ci] for a 3x3 stride-1 pad-1 conv, in torch's layout
 * [Cout, Cin, 3, 3] fp32, from the halo planes of b2s_split_halo_f16_autoscale (x [B, H+2, W+2, Cin], dout
 * [B, H+2, W+2, Cout], both halos zero), times both planes' 2^-e (x_scale_dev[0] * dout_scale_dev[0], applied as one
 * exponent).  Cin multiple of 64, Cout 64, 128 or 256.  wgmma with MN-major operands fed by TMA from the planes, 3xF16
 * (dY_hi*X_hi + dY_hi*X_lo + dY_lo*X_hi), fp32 chains of 12 MMAs drained with round-to-nearest adds.  Deterministic:
 * per-slab partials of 2048 pixels (workspace) added in slab order by a second launch, no float atomics. */
size_t b2s_conv2d_wgrad_tc_workspace_bytes(int batch, int H, int W, int Cin, int Cout);
int b2s_conv2d_wgrad_tc(const b2s_half *x_hi, const b2s_half *x_lo, const b2s_half *dout_hi, const b2s_half *dout_lo,
                        int batch, int H, int W, int Cin, int Cout, const float *x_scale_dev,
                        const float *dout_scale_dev, float *dweight, void *workspace, size_t workspace_bytes,
                        void *stream);
/* b2s_conv2d_wgrad_tc with products 3 (the same) or 1 (the f16 mode: x_lo and dout_lo NULL, one dY_hi*X_hi product per
 * tap and k16 step; a stage holds the hi planes only).  The same workspace and slab order.  The forward and the input
 * gradient of the f16 mode are b2s_conv2d_tc_ex3 launches with products = 1 and out_fp32 = 1. */
int b2s_conv2d_wgrad_tc_ex(const b2s_half *x_hi, const b2s_half *x_lo, const b2s_half *dout_hi, const b2s_half *dout_lo,
                           int batch, int H, int W, int Cin, int Cout, const float *x_scale_dev,
                           const float *dout_scale_dev, float *dweight, void *workspace, size_t workspace_bytes,
                           int products, void *stream);

/* ---- BatchNorm + ReLU in training (csrc/bn_train.cu) --------------------------------------------------------------
 * y = relu(BatchNorm(x)) as torch.nn.BatchNorm1d / BatchNorm2d.forward in train() (affine, track_running_stats, a
 * numeric momentum) followed by nn.ReLU, and its backward.  x is fp32 with `channels` channels and M = batch * spatial
 * values per channel, in one of two layouts:
 *   B2S_LAYOUT_NHWC  rows [batch * spatial, channels] (a BatchNorm1d input, or a channels_last map with spatial = H * W),
 *                    x, y, dy, dx 16-byte aligned;
 *   B2S_LAYOUT_NCHW  [batch, channels, spatial] contiguous.
 * channels a multiple of 4 in 4..1024, M >= 2, eps > 0, 0 <= momentum <= 1.
 * Forward, three kernels: float64 per-CTA sums of x - K and (x - K)^2 with K the channel's first value; one CTA adds
 * them in a fixed order into mean, the biased variance var and s = 1 / sqrt(var + eps), updates running_mean,
 * running_var (fp32, as torch's CUDA kernel: rm = momentum * mean + (1 - momentum) * rm, the variance unbiased by
 * M / (M - 1)) and num_batches_tracked (+1), and stores mu32 = fp32(mean), fp32(gamma s) and beta in the workspace; then
 * y = relu(fmaf(x - mu32, fp32(gamma s), beta)) in x's layout (y may not alias x).
 * Backward, three kernels: g = dy where that same expression is not <= 0 (torch's ReLU backward), else 0;
 * dbeta = sum g and dgamma = sum g xhat (xhat = (x - mean) s) from float64 per-CTA partials added in a fixed order;
 * dx = gamma s (g - dbeta / M - xhat dgamma / M) in float64, stored fp32 (dx NULL: only dgamma and dbeta).
 * No float atomics (two runs give the same bits), no sync (both can be captured).  workspace:
 * b2s_bn_relu_train_workspace_bytes(layout, batch, channels, spatial) (host query; 0 for a shape that is not accepted)
 * bytes, 16-byte aligned; it carries the statistics from the forward to the backward, so pass the same one to both. */
size_t b2s_bn_relu_train_workspace_bytes(int layout, int batch, int channels, int spatial);
int b2s_bn_relu_train_forward(const float *x, int layout, int batch, int channels, int spatial, const float *gamma,
                              const float *beta, float *running_mean, float *running_var, int64_t *num_batches_tracked,
                              float momentum, float eps, float *y, void *workspace, size_t workspace_bytes,
                              void *stream);
int b2s_bn_relu_train_backward(const float *x, const float *dy, int layout, int batch, int channels, int spatial,
                               const float *gamma, void *workspace, size_t workspace_bytes, float *dx, float *dgamma,
                               float *dbeta, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B2SECOND_H_ */
