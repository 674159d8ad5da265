// kitti_eval.cu -- KITTI detection formatting and evaluation on the device (see include/b2second.h):
//   b2s_kitti_convert  : lidar-frame detection records -> camera-frame KITTI rows, image-box clip, per-frame compaction
//                        (KittiDataset.convert_detection_to_kitti_annos, second/data/kitti_dataset.py:37-106)
//   b2s_kitti_overlaps : per-frame [n_dt, n_gt] overlap blocks for metric 0 (2D box), 1 (BEV), 2 (3D)
//                        (calculate_iou_partly, second/utils/eval.py:362-445, only its block diagonal)
//   b2s_kitti_eval     : ignore flags, two passes of compute_statistics_jit, get_thresholds, precision / orientation
//                        (eval_class_v3, second/utils/eval.py:479-611)
// Float64 arithmetic that the reference does in numba (no contraction) uses explicit _rn intrinsics, so the result
// does not depend on --fmad.  The rotated clip is fp32 (geometry.cuh), as the reference's numba kernel.
#include <math.h>

#include "common.cuh"
#include "geometry.cuh"

namespace {

constexpr int kSamplePts = 41;                 // N_SAMPLE_PTS of eval_class_v3
constexpr int kMaxDtPerFrame = 2048;           // assigned_detection bitmask held per thread
constexpr double kNoDetection = -10000000.0;   // NO_DETECTION of compute_statistics_jit

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

// ------------------------------------------------------------------------------------------------
// detections -> KITTI rows
// ------------------------------------------------------------------------------------------------
// one warp per frame, one lane per detection; survivors keep detection order (ballot prefix)
__global__ void k_kitti_convert(const float *__restrict__ det, int stride, int code, const int *__restrict__ det_off,
                                int F, const double *__restrict__ calib, const int *__restrict__ image_shape,
                                double *__restrict__ out, int *__restrict__ out_count)
{
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (f >= F) return;
    const double *R0 = calib + (size_t)f * 48, *Tr = R0 + 16, *P2 = R0 + 32;
    // rect @ Trv2c (lidar_to_camera, box_np_ops.py:658-663); rows 0..2 are all a point needs
    double M[12];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) s = dadd(s, dmul(R0[a * 4 + k], Tr[k * 4 + b]));
            M[a * 4 + b] = s;
        }
    const double H = (double)image_shape[2 * f], W = (double)image_shape[2 * f + 1];
    const int d0 = det_off[f], n = det_off[f + 1] - d0;
    int kept = 0;
    for (int base = 0; base < n; base += 32) {
        const int j = base + lane;
        bool keep = false;
        double row[16];
        if (j < n) {
            const float *r = det + (size_t)(d0 + j) * stride;
            const float x = r[0], y = r[1], w = r[3], l = r[4], h = r[5], ry = r[6];
            const float z = __fsub_rn(r[2], __fdiv_rn(h, 2.f));          // final_box_preds[:, 2] -= h / 2 (fp32)
            const double p[4] = {x, y, z, 1.0};
            double loc[3];
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                double s = 0.0;
#pragma unroll
                for (int b = 0; b < 4; ++b) s = dadd(s, dmul(p[b], M[a * 4 + b]));
                loc[a] = s;
            }
            // camera box (x, y, z, l, h, w, ry); corners with origin (0.5, 1, 0.5), rotated about camera y
            // (center_to_corner_box3d / rotation_3d_in_axis(axis=1), box_np_ops.py:301-319,377-402)
            const double dim[3] = {l, h, w};
            double sr, cr;
            sincos((double)ry, &sr, &cr);
            double x1 = INFINITY, y1 = INFINITY, x2 = -INFINITY, y2 = -INFINITY;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                // corners_norm order [0,1,3,2,4,5,7,6] of the (x,y,z) bit patterns
                const int bits = (c < 4) ? ((c == 2) ? 3 : (c == 3) ? 2 : c) : ((c == 6) ? 7 : (c == 7) ? 6 : c);
                const double px = dmul(dim[0], (double)((bits >> 2) & 1) - 0.5);
                const double py = dmul(dim[1], (double)((bits >> 1) & 1) - 1.0);
                const double pz = dmul(dim[2], (double)(bits & 1) - 0.5);
                const double X = dadd(dadd(dmul(px, cr), dmul(pz, sr)), loc[0]);
                const double Y = dadd(py, loc[1]);
                const double Z = dadd(dsub(dmul(pz, cr), dmul(px, sr)), loc[2]);
                // project_to_image with a zero homogeneous coordinate (box_np_ops.py:641-647)
                const double u = dadd(dadd(dmul(X, P2[0]), dmul(Y, P2[1])), dmul(Z, P2[2]));
                const double v = dadd(dadd(dmul(X, P2[4]), dmul(Y, P2[5])), dmul(Z, P2[6]));
                const double q = dadd(dadd(dmul(X, P2[8]), dmul(Y, P2[9])), dmul(Z, P2[10]));
                const double ix = u / q, iy = v / q;
                x1 = fmin(x1, ix); y1 = fmin(y1, iy); x2 = fmax(x2, ix); y2 = fmax(y2, iy);
            }
            keep = !(x1 > W || y1 > H) && !(x2 < 0.0 || y2 < 0.0);
            row[0] = fmax(x1, 0.0); row[1] = fmax(y1, 0.0); row[2] = fmin(x2, W); row[3] = fmin(y2, H);
            row[4] = loc[0]; row[5] = loc[1]; row[6] = loc[2];
            row[7] = l; row[8] = h; row[9] = w;
            row[10] = ry;
            // -arctan2(-y, x) is evaluated in fp32 by the reference (float32 box array), then widened
            row[11] = dadd((double)(-(float)atan2(-(double)y, (double)x)), (double)ry);
            row[12] = r[code];
            row[13] = 0.0;
            row[14] = 0.0;
            row[15] = r[code + 1];
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            double *o = out + (size_t)(d0 + kept + __popc(bal & ((1u << lane) - 1u))) * B2S_KITTI_ROW;
#pragma unroll
            for (int k = 0; k < 16; ++k) o[k] = row[k];
        }
        kept += __popc(bal);
    }
    if (lane == 0) out_count[f] = kept;
}

// ------------------------------------------------------------------------------------------------
// overlaps
// ------------------------------------------------------------------------------------------------
// rotated BEV intersection of two (x, y, w, l, r) boxes, zero when the stand-up boxes do not overlap
__device__ __forceinline__ float rotated_inter(const float *a5, const float *b5)
{
    float a[8], b[8], sa[4], sb[4];
    bev_corners(a5[0], a5[1], a5[2], a5[3], a5[4], a);
    bev_corners(b5[0], b5[1], b5[2], b5[3], b5[4], b);
    standup_of(a, sa);
    standup_of(b, sb);
    if (!(fminf(sa[2], sb[2]) - fmaxf(sa[0], sb[0]) > 0.f && fminf(sa[3], sb[3]) - fmaxf(sa[1], sb[1]) > 0.f))
        return 0.f;
    float area_a, area_b;
    return quad_intersection(a, b, &area_a, &area_b);
}

// one block per frame, one thread per (dt j, gt i) pair; out[ov_off[f] + j*n_gt + i]
__global__ void k_kitti_overlaps(int metric, const double *__restrict__ gt, const int *__restrict__ gt_off,
                                 const double *__restrict__ dt, const int *__restrict__ dt_off, int F,
                                 const long long *__restrict__ ov_off, int z_axis, double z_center,
                                 double *__restrict__ out)
{
    const int ax0 = 0, ax1 = (z_axis == 1) ? 2 : 1;     // the two BEV axes of location / dimensions
    for (int f = blockIdx.x; f < F; f += gridDim.x) {
        const int g0 = gt_off[f], ng = gt_off[f + 1] - g0;
        const int t0 = dt_off[f], nd = dt_off[f + 1] - t0;
        double *o = out + ov_off[f];
        for (int p = threadIdx.x; p < nd * ng; p += blockDim.x) {
            const int j = p / ng, i = p % ng;
            const double *d = dt + (size_t)(t0 + j) * B2S_KITTI_ROW, *g = gt + (size_t)(g0 + i) * B2S_KITTI_ROW;
            double r = 0.0;
            if (metric == 0) {
                // image_box_overlap(dt_boxes, gt_boxes), criterion -1 (eval.py:92-119)
                const double iw = dsub(fmin(d[2], g[2]), fmax(d[0], g[0]));
                if (iw > 0.0) {
                    const double ih = dsub(fmin(d[3], g[3]), fmax(d[1], g[1]));
                    if (ih > 0.0) {
                        const double qarea = dmul(dsub(g[2], g[0]), dsub(g[3], g[1]));
                        const double inter = dmul(iw, ih);
                        const double ua = dsub(dadd(dmul(dsub(d[2], d[0]), dsub(d[3], d[1])), qarea), inter);
                        r = inter / ua;
                    }
                }
            } else {
                // rotate_iou_gpu_eval(dt_bev, gt_bev, criterion) on fp32 (x, z, l, w, ry) boxes (eval.py:122-125,
                // 166-178); its areas are w*l products (nms_gpu.py:549-561)
                const float bd[5] = {(float)d[4 + ax0], (float)d[4 + ax1], (float)d[7 + ax0], (float)d[7 + ax1],
                                     (float)d[10]};
                const float bg[5] = {(float)g[4 + ax0], (float)g[4 + ax1], (float)g[7 + ax0], (float)g[7 + ax1],
                                     (float)g[10]};
                const float inter = rotated_inter(bg, bd);
                if (metric == 1) {
                    const float ag = __fmul_rn(bg[2], bg[3]), ad = __fmul_rn(bd[2], bd[3]);
                    r = (double)__fdiv_rn(inter, __fsub_rn(__fadd_rn(ag, ad), inter));
                } else if (inter > 0.f) {
                    // box3d_overlap_kernel (eval.py:128-164): height overlap in fp64, the ratio stored into the fp32
                    // rinc array
                    const double hd = d[7 + z_axis], hg = g[7 + z_axis], zd = d[4 + z_axis], zg = g[4 + z_axis];
                    const double max_z = fmax(dsub(zd, dmul(hd, z_center)), dsub(zg, dmul(hg, z_center)));
                    const double min_z = fmin(dadd(zd, dmul(hd, 1.0 - z_center)), dadd(zg, dmul(hg, 1.0 - z_center)));
                    const double iw = dsub(min_z, max_z);
                    if (iw > 0.0) {
                        const double area_d = dmul(dmul(d[7], d[8]), d[9]), area_g = dmul(dmul(g[7], g[8]), g[9]);
                        const double inc = dmul(iw, (double)inter);
                        r = (double)(float)(inc / dsub(dadd(area_d, area_g), inc));
                    }
                }
            }
            o[(size_t)j * ng + i] = r;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// evaluation
// ------------------------------------------------------------------------------------------------
struct Task {
    int cls, alt, difficulty;   // class vocabulary id; id that counts as "valid 0" (Van / Person_sitting) or -3
    double min_overlap;
};

__device__ __forceinline__ Task load_task(const int *task_info, const double *task_min_overlap, int t)
{
    return Task{task_info[3 * t], task_info[3 * t + 1], task_info[3 * t + 2], task_min_overlap[t]};
}

// clean_data (eval.py:33-89) for every (task, box): ignored_gt / ignored_dt in {-1, 0, 1}; num_valid_gt per task.
// Whether a box lies outside the task's difficulty (height, truncation, occlusion) is bit `difficulty` of its limits
// byte: the host takes those comparisons in the annotation's own dtype, as the reference does.
__global__ void k_kitti_clean(const int *__restrict__ gt_name, const uint8_t *__restrict__ gt_limits, int G,
                              const int *__restrict__ dt_name, const uint8_t *__restrict__ dt_limits, int D,
                              const int *__restrict__ task_info, const double *__restrict__ task_min_overlap, int T,
                              int8_t *__restrict__ ign_gt, int8_t *__restrict__ ign_dt, int *__restrict__ num_valid)
{
    const long long total = (long long)T * (G + D);
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total;
         g += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(g / (G + D)), k = (int)(g % (G + D));
        const Task task = load_task(task_info, task_min_overlap, t);
        const int diff = task.difficulty;
        if (k < G) {
            const int name = gt_name[k];
            const int valid = (name == task.cls) ? 1 : (name == task.alt) ? 0 : -1;
            const bool ignore = (gt_limits[k] >> diff) & 1;
            int8_t v;
            if (valid == 1 && !ignore) {
                v = 0;
                atomicAdd(&num_valid[t], 1);
            } else if (valid == 0 || (ignore && valid == 1)) {
                v = 1;
            } else {
                v = -1;
            }
            ign_gt[(size_t)t * G + k] = v;
        } else {
            const int j = k - G;
            ign_dt[(size_t)t * D + j] = ((dt_limits[j] >> diff) & 1) ? 1 : (dt_name[j] == task.cls) ? 0 : -1;
        }
    }
}

struct Stats {
    int tp, fp;
    double similarity;   // 0 when the reference returns -1 (nothing to add)
};

// compute_statistics_jit (eval.py:181-300) for one frame.  compute_fp = false: the true positives' scores go to
// tp_scores (gt order).  Matching order and tie rules are the reference's: gts in order, dets in order, strict >.
__device__ Stats frame_statistics(const double *__restrict__ ov, const double *__restrict__ gt, const int *gt_name,
                                  int ng, const double *__restrict__ dt, int nd, const int8_t *__restrict__ ign_gt,
                                  const int8_t *__restrict__ ign_dt, int metric, double min_overlap, double thresh,
                                  bool compute_fp, bool compute_aos, double *tp_scores)
{
    unsigned assigned[kMaxDtPerFrame / 32];
    const int words = (nd + 31) >> 5;
    for (int w = 0; w < words; ++w) assigned[w] = 0u;
    auto is_assigned = [&](int j) { return (assigned[j >> 5] >> (j & 31)) & 1u; };
    auto assign = [&](int j) { assigned[j >> 5] |= 1u << (j & 31); };
    auto below = [&](int j) { return compute_fp && dt[(size_t)j * B2S_KITTI_ROW + 12] < thresh; };
    Stats s{0, 0, 0.0};
    for (int i = 0; i < ng; ++i) {
        const int ig = ign_gt[i];
        if (ig == -1) continue;
        int det_idx = -1;
        double valid_detection = kNoDetection, max_overlap = 0.0;
        bool assigned_ignored_det = false;
        for (int j = 0; j < nd; ++j) {
            const int id = ign_dt[j];
            if (id == -1 || is_assigned(j) || below(j)) continue;
            const double overlap = ov[(size_t)j * ng + i];
            const double dt_score = dt[(size_t)j * B2S_KITTI_ROW + 12];
            if (!compute_fp && overlap > min_overlap && dt_score > valid_detection) {
                det_idx = j;
                valid_detection = dt_score;
            } else if (compute_fp && overlap > min_overlap && (overlap > max_overlap || assigned_ignored_det) &&
                       id == 0) {
                max_overlap = overlap;
                det_idx = j;
                valid_detection = 1.0;
                assigned_ignored_det = false;
            } else if (compute_fp && overlap > min_overlap && valid_detection == kNoDetection && id == 1) {
                det_idx = j;
                valid_detection = 1.0;
                assigned_ignored_det = true;
            }
        }
        if (valid_detection == kNoDetection) continue;   // fn (not needed by the precision)
        if (ig == 1 || ign_dt[det_idx] == 1) {
            assign(det_idx);
        } else {
            if (tp_scores) tp_scores[s.tp] = dt[(size_t)det_idx * B2S_KITTI_ROW + 12];
            ++s.tp;
            if (compute_aos) {
                // sequential np.sum over fp zeros then the deltas in gt order
                const double delta = dsub(gt[(size_t)i * B2S_KITTI_ROW + 11], dt[(size_t)det_idx * B2S_KITTI_ROW + 11]);
                s.similarity = dadd(s.similarity, dadd(1.0, cos(delta)) / 2.0);
            }
            assign(det_idx);
        }
    }
    if (compute_fp) {
        for (int j = 0; j < nd; ++j)
            if (!(is_assigned(j) || ign_dt[j] == -1 || ign_dt[j] == 1 || below(j))) ++s.fp;
        if (metric == 0) {
            // don't-care boxes: image_box_overlap(dt_bboxes, dc_bboxes, criterion 0) (eval.py:273-287)
            int nstuff = 0;
            for (int i = 0; i < ng; ++i) {
                if (gt_name[i] != B2S_KITTI_DONTCARE) continue;
                const double *c = gt + (size_t)i * B2S_KITTI_ROW;
                for (int j = 0; j < nd; ++j) {
                    if (is_assigned(j) || ign_dt[j] == -1 || ign_dt[j] == 1 || below(j)) continue;
                    const double *d = dt + (size_t)j * B2S_KITTI_ROW;
                    double o = 0.0;
                    const double iw = dsub(fmin(d[2], c[2]), fmax(d[0], c[0]));
                    if (iw > 0.0) {
                        const double ih = dsub(fmin(d[3], c[3]), fmax(d[1], c[1]));
                        if (ih > 0.0) o = dmul(iw, ih) / dmul(dsub(d[2], d[0]), dsub(d[3], d[1]));
                    }
                    if (o > min_overlap) {
                        assign(j);
                        ++nstuff;
                    }
                }
            }
            s.fp -= nstuff;
        }
    }
    return s;
}

// pass 1: one thread per (task, frame); tp scores land in the frame's gt slots, the rest of the slots get -inf
__global__ void k_kitti_pass1(int metric, const double *__restrict__ gt, const int *__restrict__ gt_name,
                              const int *__restrict__ gt_off, int G, const double *__restrict__ dt,
                              const int *__restrict__ dt_off, int D, int F, const double *__restrict__ ov,
                              const long long *__restrict__ ov_off, const double *__restrict__ task_min_overlap, int T,
                              const int8_t *__restrict__ ign_gt, const int8_t *__restrict__ ign_dt, int Gp,
                              double *__restrict__ scores, int *__restrict__ tp_total)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)T * F) return;
    const int t = (int)(g / F), f = (int)(g % F);
    const int g0 = gt_off[f], ng = gt_off[f + 1] - g0, d0 = dt_off[f], nd = dt_off[f + 1] - d0;
    double *out = scores + (size_t)t * Gp + g0;
    const Stats s = frame_statistics(ov + ov_off[f], gt + (size_t)g0 * B2S_KITTI_ROW, gt_name + g0, ng,
                                     dt + (size_t)d0 * B2S_KITTI_ROW, nd, ign_gt + (size_t)t * G + g0,
                                     ign_dt + (size_t)t * D + d0, metric, task_min_overlap[t], 0.0, false, false, out);
    for (int k = s.tp; k < ng; ++k) out[k] = -INFINITY;
    if (s.tp) atomicAdd(&tp_total[t], s.tp);
}

// one block per task: bitonic sort of the Gp score slots (descending, in global memory), then get_thresholds
// (eval.py:11-30) on one thread
__global__ void k_kitti_thresholds(int G, int Gp, double *__restrict__ scores, const int *__restrict__ tp_total,
                                   const int *__restrict__ num_valid, double *__restrict__ thr, int *__restrict__ nthr)
{
    const int t = blockIdx.x;
    double *s = scores + (size_t)t * Gp;
    for (int k = G + threadIdx.x; k < Gp; k += blockDim.x) s[k] = -INFINITY;
    __syncthreads();
    for (int size = 2; size <= Gp; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int idx = threadIdx.x; idx < (Gp >> 1); idx += blockDim.x) {
                const int lo = 2 * stride * (idx / stride) + idx % stride, hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const double a = s[lo], b = s[hi];
                if ((a < b) == desc && a != b) { s[lo] = b; s[hi] = a; }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x != 0) return;
    const int n = tp_total[t];
    const double num_gt = (double)num_valid[t];
    double current_recall = 0.0;
    int cnt = 0;
    for (int i = 0; i < n; ++i) {
        const double l_recall = (double)(i + 1) / num_gt;
        const double r_recall = (i < n - 1) ? (double)(i + 2) / num_gt : l_recall;
        if (dsub(r_recall, current_recall) < dsub(current_recall, l_recall) && i < n - 1) continue;
        if (cnt < kSamplePts) thr[t * kSamplePts + cnt] = s[i];
        ++cnt;
        current_recall = dadd(current_recall, 1.0 / (kSamplePts - 1.0));
    }
    nthr[t] = cnt < kSamplePts ? cnt : kSamplePts;
}

// pass 2: one thread per (task, frame, threshold)
__global__ void k_kitti_pass2(int metric, const double *__restrict__ gt, const int *__restrict__ gt_name,
                              const int *__restrict__ gt_off, int G, const double *__restrict__ dt,
                              const int *__restrict__ dt_off, int D, int F, const double *__restrict__ ov,
                              const long long *__restrict__ ov_off, const double *__restrict__ task_min_overlap, int T,
                              const int8_t *__restrict__ ign_gt, const int8_t *__restrict__ ign_dt,
                              const double *__restrict__ thr, const int *__restrict__ nthr, int compute_aos,
                              int2 *__restrict__ counts, double *__restrict__ sims)
{
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= (long long)T * F * kSamplePts) return;
    const int k = (int)(g % kSamplePts);
    const long long tf = g / kSamplePts;
    const int t = (int)(tf / F), f = (int)(tf % F);
    if (k >= nthr[t]) return;
    const int g0 = gt_off[f], ng = gt_off[f + 1] - g0, d0 = dt_off[f], nd = dt_off[f + 1] - d0;
    const Stats s = frame_statistics(ov + ov_off[f], gt + (size_t)g0 * B2S_KITTI_ROW, gt_name + g0, ng,
                                     dt + (size_t)d0 * B2S_KITTI_ROW, nd, ign_gt + (size_t)t * G + g0,
                                     ign_dt + (size_t)t * D + d0, metric, task_min_overlap[t],
                                     thr[t * kSamplePts + k], true, compute_aos != 0, nullptr);
    const size_t o = ((size_t)t * kSamplePts + k) * F + f;
    counts[o] = make_int2(s.tp, s.fp);
    sims[o] = s.similarity;
}

__device__ __forceinline__ double nan_max(double m, double v) { return (isnan(m) || isnan(v)) ? NAN : fmax(m, v); }

// one block per task: frame-ordered sums (pr[t, :] of eval_class_v3), precision / orientation, running max from the
// right (eval.py:581-591)
__global__ void k_kitti_finalize(int F, const int2 *__restrict__ counts, const double *__restrict__ sims,
                                 const double *__restrict__ thr, const int *__restrict__ nthr, int compute_aos,
                                 double *__restrict__ precision, double *__restrict__ orientation,
                                 double *__restrict__ thresholds)
{
    __shared__ double s_prec[kSamplePts], s_aos[kSamplePts];
    const int t = blockIdx.x, k = threadIdx.x, n = nthr[t];
    if (k < kSamplePts) {
        double tp = 0.0, fp = 0.0, sim = 0.0;
        if (k < n) {
            const size_t o = ((size_t)t * kSamplePts + k) * F;
            for (int f = 0; f < F; ++f) {
                const int2 c = counts[o + f];
                tp = dadd(tp, (double)c.x);
                fp = dadd(fp, (double)c.y);
                sim = dadd(sim, sims[o + f]);
            }
        }
        s_prec[k] = k < n ? tp / dadd(tp, fp) : 0.0;
        s_aos[k] = (k < n && compute_aos) ? sim / dadd(tp, fp) : 0.0;
        thresholds[t * kSamplePts + k] = k < n ? thr[t * kSamplePts + k] : 0.0;
    }
    __syncthreads();
    if (k != 0) return;
    double mp = 0.0, ma = 0.0;
    for (int i = kSamplePts - 1; i >= 0; --i) {
        if (i < n) {
            mp = nan_max(mp, s_prec[i]);
            ma = nan_max(ma, s_aos[i]);
            s_prec[i] = mp;
            s_aos[i] = ma;
        }
        precision[t * kSamplePts + i] = s_prec[i];
        orientation[t * kSamplePts + i] = s_aos[i];
    }
}

int next_pow2(int x)
{
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

struct EvalWorkspace {
    int8_t *ign_gt, *ign_dt;
    int *num_valid, *tp_total, *nthr;
    double *scores, *thr, *sims;
    int2 *counts;
    size_t bytes;
};

EvalWorkspace carve(char *base, int F, int G, int D, int T)
{
    EvalWorkspace w;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        char *p = base ? base + off : nullptr;
        off += b2s_align(bytes);
        return p;
    };
    w.num_valid = (int *)take(sizeof(int) * 3 * (size_t)T);   // num_valid, tp_total, nthr: one memset
    w.tp_total = w.num_valid ? w.num_valid + T : nullptr;
    w.nthr = w.num_valid ? w.num_valid + 2 * T : nullptr;
    w.ign_gt = (int8_t *)take((size_t)T * G);
    w.ign_dt = (int8_t *)take((size_t)T * D);
    w.scores = (double *)take(sizeof(double) * (size_t)T * next_pow2(G > 0 ? G : 1));
    w.thr = (double *)take(sizeof(double) * (size_t)T * kSamplePts);
    w.counts = (int2 *)take(sizeof(int2) * (size_t)T * kSamplePts * F);
    w.sims = (double *)take(sizeof(double) * (size_t)T * kSamplePts * F);
    w.bytes = off;
    return w;
}

}  // namespace

extern "C" int b2s_kitti_convert(const float *det, int det_stride, int code, const int *det_off, int num_frames,
                                 const double *calib, const int *image_shape, double *out, int *out_count_dev,
                                 void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(num_frames >= 0 && code >= 7 && det_stride >= code + 2, "b2s_kitti_convert: bad arguments");
    if (num_frames == 0) return 0;
    k_kitti_convert<<<b2s_cdiv(num_frames, 4), 128, 0, stream>>>(det, det_stride, code, det_off, num_frames, calib,
                                                                 image_shape, out, out_count_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_kitti_overlaps(int metric, const double *gt, const int *gt_off, const double *dt, const int *dt_off,
                                  int num_frames, const long long *ov_off, int z_axis, double z_center, double *out,
                                  void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(metric >= 0 && metric <= 2 && num_frames >= 0 && (z_axis == 1 || z_axis == 2),
                "b2s_kitti_overlaps: bad arguments (metric 0..2, z_axis 1 or 2)");
    if (num_frames == 0) return 0;
    const int blocks = num_frames < 132 * 16 ? num_frames : 132 * 16;
    k_kitti_overlaps<<<blocks, 128, 0, stream>>>(metric, gt, gt_off, dt, dt_off, num_frames, ov_off, z_axis, z_center,
                                                 out);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" size_t b2s_kitti_eval_workspace_bytes(int num_frames, int num_gt, int num_dt, int num_tasks)
{
    return carve(nullptr, num_frames, num_gt, num_dt, num_tasks).bytes;
}

extern "C" int b2s_kitti_eval(int metric, const double *gt, const int *gt_name, const uint8_t *gt_limits,
                              const int *gt_off, int num_gt, const double *dt, const int *dt_name,
                              const uint8_t *dt_limits, const int *dt_off, int num_dt, int num_frames,
                              int max_dt_per_frame, const double *overlaps, const long long *ov_off,
                              const int *task_info, const double *task_min_overlap, int num_tasks, int compute_aos,
                              double *precision, double *orientation, double *thresholds, void *workspace,
                              size_t workspace_bytes, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(metric >= 0 && metric <= 2 && num_frames >= 1 && num_gt >= 0 && num_dt >= 0 && num_tasks >= 0,
                "b2s_kitti_eval: bad arguments");
    B2S_REQUIRE(max_dt_per_frame <= kMaxDtPerFrame, "b2s_kitti_eval: %d detections in one frame (at most %d)",
                max_dt_per_frame, kMaxDtPerFrame);
    B2S_REQUIRE((num_gt == 0 || gt_limits != nullptr) && (num_dt == 0 || dt_limits != nullptr),
                "b2s_kitti_eval: gt_limits / dt_limits (difficulty limit bits) are required");
    if (num_tasks == 0) return 0;
    const int F = num_frames, G = num_gt, D = num_dt, T = num_tasks, Gp = next_pow2(G > 0 ? G : 1);
    EvalWorkspace w = carve((char *)workspace, F, G, D, T);
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= w.bytes, "b2s_kitti_eval: workspace too small");
    B2S_CUDA_OK(cudaMemsetAsync(w.num_valid, 0, sizeof(int) * 3 * (size_t)T, stream));
    if (G + D > 0) {
        long long total = (long long)T * (G + D);
        int blocks = b2s_cdiv(total, 256);
        if (blocks > 132 * 16) blocks = 132 * 16;
        k_kitti_clean<<<blocks, 256, 0, stream>>>(gt_name, gt_limits, G, dt_name, dt_limits, D, task_info,
                                                  task_min_overlap, T, w.ign_gt, w.ign_dt, w.num_valid);
        B2S_LAUNCH_OK();
    }
    k_kitti_pass1<<<b2s_cdiv((long long)T * F, 128), 128, 0, stream>>>(
        metric, gt, gt_name, gt_off, G, dt, dt_off, D, F, overlaps, ov_off, task_min_overlap, T, w.ign_gt, w.ign_dt, Gp,
        w.scores, w.tp_total);
    B2S_LAUNCH_OK();
    k_kitti_thresholds<<<T, 1024, 0, stream>>>(G, Gp, w.scores, w.tp_total, w.num_valid, w.thr, w.nthr);
    B2S_LAUNCH_OK();
    k_kitti_pass2<<<b2s_cdiv((long long)T * F * kSamplePts, 128), 128, 0, stream>>>(
        metric, gt, gt_name, gt_off, G, dt, dt_off, D, F, overlaps, ov_off, task_min_overlap, T, w.ign_gt, w.ign_dt,
        w.thr, w.nthr, compute_aos, w.counts, w.sims);
    B2S_LAUNCH_OK();
    k_kitti_finalize<<<T, 64, 0, stream>>>(F, w.counts, w.sims, w.thr, w.nthr, compute_aos, precision, orientation,
                                           thresholds);
    B2S_LAUNCH_OK();
    return 0;
}
