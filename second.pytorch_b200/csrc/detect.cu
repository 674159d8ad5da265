// detect.cu -- SECOND predict step on the device (see include/b2second.h):
//   b2s_decode_filter : box decode + sigmoid + score threshold over all anchors -> candidate list
//                       (_strided: any head layout; _segments: several head maps into one list per frame)
//   b2s_nms           : deterministic top-k (score desc, anchor asc) -> pairwise IoU bitmask
//                       (rotated polygon clip, or stand-up boxes with the +1 convention)
//                       -> greedy reduce in shared memory -> direction fix-up + range test
//   b2s_nms_*_host    : numpy-facing spconv.utils signatures
// Nothing here synchronises with the host (except the *_host wrappers, by contract).
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "geometry.cuh"

namespace {

constexpr int kSortCap = 4096;     // bitonic sort capacity (keys in shared memory)
constexpr int kSelThreads = 1024;
constexpr int kMaxCode = 16;

// ------------------------------------------------------------------------------------------------
// decode + filter
// ------------------------------------------------------------------------------------------------
// head element (b, channel ch, pixel hw) lives at t[b*batch_stride + ch*cs + hw*ps]
struct HeadStrides {
    long long box_b, cls_b, dir_b;
    int cs, ps;
};

// one anchor: score = max over classes of the sigmoid (first class wins ties), threshold, append to frame b's list
__device__ __forceinline__ void decode_filter_one(const float *__restrict__ box, const float *__restrict__ cls,
                                                  const float *__restrict__ dir, const HeadStrides &hs,
                                                  const float *__restrict__ an, int b, int al, int hw, int anchor_id,
                                                  int code, int ncls, int nbins, float thresh, float *cand_box,
                                                  float *cand_score, int *cand_label, int *cand_dir, int *cand_anchor,
                                                  int *cand_count, int cand_cap, unsigned *status)
{
    const size_t cs = (size_t)hs.cs, ps = (size_t)hs.ps;
    // class scores: the reference takes max/argmax over the SIGMOID scores (voxelnet.py:444,554-555), so
    // saturated or fp32-equal scores tie and the first class wins -- compare scores, not logits.
    const float *cp = cls + (size_t)b * hs.cls_b + (size_t)al * ncls * cs + (size_t)hw * ps;
    float score = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-__ldg(cp))));
    int label = 0;
    for (int c = 1; c < ncls; ++c) {
        float s = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-__ldg(cp + (size_t)c * cs))));
        if (s > score) { score = s; label = c; }
    }
    if (!(score >= thresh)) return;
    int pos = atomicAdd(&cand_count[b], 1);
    if (pos >= cand_cap) { atomicOr(status, B2S_STATUS_CAND_OVERFLOW); return; }
    const size_t slot = (size_t)b * cand_cap + pos;
    // box decode (second_box_decode): separate mul/add like the elementwise reference ops
    const float *bp = box + (size_t)b * hs.box_b + (size_t)al * code * cs + (size_t)hw * ps;
    float t[kMaxCode], q[kMaxCode];
    for (int i = 0; i < code; ++i) { t[i] = __ldg(bp + (size_t)i * cs); q[i] = __ldg(&an[i]); }
    const float xa = q[0], ya = q[1], za = q[2], wa = q[3], la = q[4], ha = q[5], ra = q[6];
    const float diag = sqrtf(__fadd_rn(__fmul_rn(la, la), __fmul_rn(wa, wa)));
    float o[kMaxCode];
    o[0] = __fadd_rn(__fmul_rn(t[0], diag), xa);
    o[1] = __fadd_rn(__fmul_rn(t[1], diag), ya);
    o[2] = __fadd_rn(__fmul_rn(t[2], ha), za);
    o[3] = __fmul_rn(expf(t[3]), wa);
    o[4] = __fmul_rn(expf(t[4]), la);
    o[5] = __fmul_rn(expf(t[5]), ha);
    o[6] = __fadd_rn(t[6], ra);
    for (int i = 7; i < code; ++i) o[i] = __fadd_rn(t[i], q[i]);
    float *cb = cand_box + slot * code;
    for (int i = 0; i < code; ++i) cb[i] = o[i];
    cand_score[slot] = score;
    cand_label[slot] = label;
    int dl = 0;
    if (dir != nullptr) {
        const float *dp = dir + (size_t)b * hs.dir_b + (size_t)al * nbins * cs + (size_t)hw * ps;
        float bd = __ldg(dp);
        for (int c = 1; c < nbins; ++c) {
            float v = __ldg(dp + (size_t)c * cs);
            if (v > bd) { bd = v; dl = c; }
        }
    }
    cand_dir[slot] = dl;
    cand_anchor[slot] = anchor_id;
}

__global__ void k_decode_filter(const float *__restrict__ box, const float *__restrict__ cls,
                                const float *__restrict__ dir, HeadStrides hs, const float *__restrict__ anchors,
                                const uint8_t *__restrict__ amask, int batch, int a_loc, int H, int W,
                                int code, int ncls, int nbins, float thresh, float *cand_box,
                                float *cand_score, int *cand_label, int *cand_dir, int *cand_anchor,
                                int *cand_count, int cand_cap, unsigned *status)
{
    const int HW = H * W;
    const int A = a_loc * HW;
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)batch * A) return;
    const int b = (int)(gid / A), a = (int)(gid % A);
    if (amask != nullptr && amask[gid] == 0) return;
    decode_filter_one(box, cls, dir, hs, anchors + (size_t)a * code, b, a / HW, a % HW, a, code, ncls, nbins, thresh,
                      cand_box, cand_score, cand_label, cand_dir, cand_anchor, cand_count, cand_cap, status);
}

// several head maps (b2s_decode_filter_segments): segment s owns the global anchors [base_s, base_s + a_loc_s*H_s*W_s)
struct Segments {
    const float *box[B2S_MAX_HEAD_SEGMENTS], *cls[B2S_MAX_HEAD_SEGMENTS], *dir[B2S_MAX_HEAD_SEGMENTS];
    HeadStrides hs[B2S_MAX_HEAD_SEGMENTS];
    int a_loc[B2S_MAX_HEAD_SEGMENTS], H[B2S_MAX_HEAD_SEGMENTS], W[B2S_MAX_HEAD_SEGMENTS];
    int base[B2S_MAX_HEAD_SEGMENTS];
    int n;
};

__global__ void k_decode_filter_segments(Segments sg, const float *__restrict__ anchors,
                                         const uint8_t *__restrict__ amask, int batch, int num_anchors, int code,
                                         int ncls, int nbins, float thresh, float *cand_box, float *cand_score,
                                         int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count,
                                         int cand_cap, unsigned *status)
{
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)batch * num_anchors) return;
    const int b = (int)(gid / num_anchors), a = (int)(gid % num_anchors);
    if (amask != nullptr && amask[gid] == 0) return;
    int s = -1;
#pragma unroll
    for (int i = 0; i < B2S_MAX_HEAD_SEGMENTS; ++i)
        if (i < sg.n && a >= sg.base[i] && a - sg.base[i] < sg.a_loc[i] * sg.H[i] * sg.W[i]) s = i;
    if (s < 0) return;                                   // an anchor no segment covers (gaps are allowed)
    const int HW = sg.H[s] * sg.W[s];
    const int al = (a - sg.base[s]) / HW, hw = (a - sg.base[s]) % HW;
    decode_filter_one(sg.box[s], sg.cls[s], sg.dir[s], sg.hs[s], anchors + (size_t)a * code, b, al, hw, a, code, ncls,
                      nbins, thresh, cand_box, cand_score, cand_label, cand_dir, cand_anchor, cand_count, cand_cap,
                      status);
}

// Per-class variant for the multi-class NMS branch (voxelnet.py:458-547): one candidate list per (class, frame) --
// "virtual frame" v = c*batch + b, class-major so that one class's frames are contiguous.  An anchor joins class c's
// list when its class-c sigmoid score passes that class's threshold and (unless class-agnostic) the anchor belongs
// to class c's anchor range [cls_lo[c], cls_hi[c]) of a_loc indices (target_assigner.anchors_range).  The label of
// every candidate of list (c, b) is c.
struct ClassRanges {
    int lo[16], hi[16];
    float thresh[16];
};

__global__ void k_decode_filter_mc(const float *__restrict__ box, const float *__restrict__ cls,
                                   const float *__restrict__ dir, HeadStrides hs, const float *__restrict__ anchors,
                                   int batch, int a_loc, int H, int W, int code, int ncls, int nbins, ClassRanges cr,
                                   float *cand_box, float *cand_score, int *cand_label, int *cand_dir,
                                   int *cand_anchor, int *cand_count, int cand_cap, unsigned *status)
{
    const int HW = H * W;
    const int A = a_loc * HW;
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (long long)batch * A) return;
    const int b = (int)(gid / A), a = (int)(gid % A);
    const int al = a / HW, hw = a % HW;
    const size_t cs = (size_t)hs.cs, ps = (size_t)hs.ps;
    const float *cp = cls + (size_t)b * hs.cls_b + (size_t)al * ncls * cs + (size_t)hw * ps;
    bool decoded = false;
    float o[kMaxCode];
    int dl = 0;
    for (int c = 0; c < ncls; ++c) {
        if (al < cr.lo[c] || al >= cr.hi[c]) continue;
        const float score = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-__ldg(cp + (size_t)c * cs))));
        if (!(score >= cr.thresh[c])) continue;
        if (!decoded) {
            const float *bp = box + (size_t)b * hs.box_b + (size_t)al * code * cs + (size_t)hw * ps;
            const float *an = anchors + (size_t)a * code;
            float t[kMaxCode], q[kMaxCode];
            for (int i = 0; i < code; ++i) { t[i] = __ldg(bp + (size_t)i * cs); q[i] = __ldg(&an[i]); }
            const float diag = sqrtf(__fadd_rn(__fmul_rn(q[4], q[4]), __fmul_rn(q[3], q[3])));
            o[0] = __fadd_rn(__fmul_rn(t[0], diag), q[0]);
            o[1] = __fadd_rn(__fmul_rn(t[1], diag), q[1]);
            o[2] = __fadd_rn(__fmul_rn(t[2], q[5]), q[2]);
            o[3] = __fmul_rn(expf(t[3]), q[3]);
            o[4] = __fmul_rn(expf(t[4]), q[4]);
            o[5] = __fmul_rn(expf(t[5]), q[5]);
            o[6] = __fadd_rn(t[6], q[6]);
            for (int i = 7; i < code; ++i) o[i] = __fadd_rn(t[i], q[i]);
            if (dir != nullptr) {
                const float *dp = dir + (size_t)b * hs.dir_b + (size_t)al * nbins * cs + (size_t)hw * ps;
                float bd = __ldg(dp);
                for (int k = 1; k < nbins; ++k) {
                    float v = __ldg(dp + (size_t)k * cs);
                    if (v > bd) { bd = v; dl = k; }
                }
            }
            decoded = true;
        }
        const int v = c * batch + b;
        int pos = atomicAdd(&cand_count[v], 1);
        if (pos >= cand_cap) { atomicOr(status, B2S_STATUS_CAND_OVERFLOW); continue; }
        const size_t slot = (size_t)v * cand_cap + pos;
        float *cb = cand_box + slot * code;
        for (int i = 0; i < code; ++i) cb[i] = o[i];
        cand_score[slot] = score;
        cand_label[slot] = c;
        cand_dir[slot] = dl;
        cand_anchor[slot] = a;
    }
}

// concatenate the per-class NMS results of one frame in class order (voxelnet.py:528-533): in [ncls*B, post_max, S]
// + counts [ncls*B] (class-major) -> record b: rows, then (det_frame_stride > rows*S) the count as a float
__global__ void k_concat_classes(const float *__restrict__ det_mc, const int *__restrict__ cnt_mc, int batch, int ncls,
                                 int post_max, int S, float *det, int det_frame_stride, int *det_count)
{
    const int b = blockIdx.x;
    __shared__ int s_off[17];
    if (threadIdx.x == 0) {
        int off = 0;
        for (int c = 0; c < ncls; ++c) { s_off[c] = off; off += min(cnt_mc[c * batch + b], post_max); }
        s_off[ncls] = off;
        det_count[b] = off;
        if (det_frame_stride > ncls * post_max * S) det[(size_t)b * det_frame_stride + det_frame_stride - 1] = (float)off;
    }
    __syncthreads();
    for (int c = 0; c < ncls; ++c) {
        const int n = s_off[c + 1] - s_off[c];
        const float *src = det_mc + (size_t)(c * batch + b) * post_max * S;
        float *dst = det + (size_t)b * det_frame_stride + (size_t)s_off[c] * S;
        for (int i = threadIdx.x; i < n * S; i += blockDim.x) dst[i] = src[i];
    }
}

__device__ __forceinline__ bool suppress_rotated(const float *ci, const float *si, const float *cj,
                                                 const float *sj, float thresh)
{
    // stand-up IoU (eps=0) must be > 0: both overlaps strictly positive
    float iw = fminf(si[2], sj[2]) - fmaxf(si[0], sj[0]);
    float ih = fminf(si[3], sj[3]) - fmaxf(si[1], sj[1]);
    if (!(iw > 0.f && ih > 0.f)) return false;
    float sa, sb;
    float inter = quad_intersection(ci, cj, &sa, &sb);
    if (!(inter > 0.f)) return false;
    float iou = inter / (sa + sb - inter);
    return iou >= thresh;
}

// eps = 1, inclusive = false : spconv.utils.non_max_suppression (Fast-R-CNN "+1", suppress if IoU >  thresh)
// eps given, inclusive = true : spconv.utils.non_max_suppression_cpu           (suppress if IoU >= thresh)
__device__ __forceinline__ bool suppress_aligned(const float *a, const float *b, float thresh, float eps,
                                                 bool inclusive)
{
    float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    float width = fmaxf(right - left + eps, 0.f), height = fmaxf(bottom - top + eps, 0.f);
    float interS = width * height;
    float Sa = (a[2] - a[0] + eps) * (a[3] - a[1] + eps);
    float Sb = (b[2] - b[0] + eps) * (b[3] - b[1] + eps);
    float iou = interS / (Sa + Sb - interS);
    if (inclusive) return (width > 0.f && height > 0.f) && iou >= thresh;
    return iou > thresh;
}

// ------------------------------------------------------------------------------------------------
// top-k select + sort: one CTA per frame
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long make_key(float score, int anchor)
{
    return ((unsigned long long)__float_as_uint(score) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)anchor);
}

// geo layout per sorted box: corners[8] + standup[4] = 12 floats
__global__ void __launch_bounds__(kSelThreads)
k_select_sort(const float *__restrict__ cand_box, const float *__restrict__ cand_score,
              const int *__restrict__ cand_anchor, const int *__restrict__ cand_count, int cand_cap, int code,
              int pre_max, int *sorted_slot /*[B,pre_max]*/, float *geo /*[B,pre_max,12]*/,
              int *n_sorted /*[B]*/)
{
    extern __shared__ __align__(16) unsigned char sm[];
    unsigned long long *s_key = reinterpret_cast<unsigned long long *>(sm);  // [kSortCap]
    int *s_slot = reinterpret_cast<int *>(s_key + kSortCap);                 // [kSortCap]
    __shared__ int s_hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_remaining, s_fill;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int nc = min(cand_count[b], cand_cap);
    const float *sc = cand_score + (size_t)b * cand_cap;
    const int *an = cand_anchor + (size_t)b * cand_cap;
    int m;  // number of keys staged in shared memory
    if (nc <= kSortCap) {
        for (int i = tid; i < kSortCap; i += kSelThreads) {
            if (i < nc) { s_key[i] = make_key(sc[i], an[i]); s_slot[i] = i; }
            else { s_key[i] = 0ull; s_slot[i] = -1; }
        }
        m = nc;
        __syncthreads();
    } else {
        // radix select (MSB first, 8 bits per pass) of the pre_max-th largest key
        const int k = min(pre_max, nc);
        if (tid == 0) { s_prefix = 0ull; s_remaining = k; }
        __syncthreads();
        for (int shift = 56; shift >= 0; shift -= 8) {
            if (tid < 256) s_hist[tid] = 0;
            __syncthreads();
            const unsigned long long prefix = s_prefix;
            const unsigned long long himask = (shift == 56) ? 0ull : (~0ull << (shift + 8));
            for (int i = tid; i < nc; i += kSelThreads) {
                unsigned long long key = make_key(sc[i], an[i]);
                if ((key & himask) == prefix) atomicAdd(&s_hist[(int)((key >> shift) & 0xFF)], 1);
            }
            __syncthreads();
            if (tid == 0) {
                int rem = s_remaining, d = 255;
                for (; d > 0; --d) {
                    if (s_hist[d] >= rem) break;
                    rem -= s_hist[d];
                }
                s_prefix = prefix | ((unsigned long long)d << shift);
                s_remaining = rem;
            }
            __syncthreads();
        }
        const unsigned long long kth = s_prefix;  // exact k-th largest key (keys are unique)
        if (tid == 0) s_fill = 0;
        __syncthreads();
        for (int i = tid; i < kSortCap; i += kSelThreads) { s_key[i] = 0ull; s_slot[i] = -1; }
        __syncthreads();
        for (int i = tid; i < nc; i += kSelThreads) {
            unsigned long long key = make_key(sc[i], an[i]);
            if (key >= kth) {
                int p = atomicAdd(&s_fill, 1);
                if (p < kSortCap) { s_key[p] = key; s_slot[p] = i; }
            }
        }
        __syncthreads();
        m = min(s_fill, kSortCap);
    }
    // bitonic sort, descending, kSortCap elements (zero keys sink to the end)
    for (int size = 2; size <= kSortCap; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < kSortCap / 2; i += kSelThreads) {
                int lo = 2 * i - (i & (stride - 1));
                int hi = lo + stride;
                bool desc = ((lo & size) == 0);
                unsigned long long a = s_key[lo], c = s_key[hi];
                bool swap = desc ? (a < c) : (a > c);
                if (swap) {
                    s_key[lo] = c; s_key[hi] = a;
                    int t = s_slot[lo]; s_slot[lo] = s_slot[hi]; s_slot[hi] = t;
                }
            }
            __syncthreads();
        }
    }
    const int n = min(m, pre_max);
    if (tid == 0) n_sorted[b] = n;
    for (int i = tid; i < n; i += kSelThreads) {
        int slot = s_slot[i];
        sorted_slot[(size_t)b * pre_max + i] = slot;
        const float *bx = cand_box + ((size_t)b * cand_cap + slot) * code;
        float c[8], s4[4];
        bev_corners(bx[0], bx[1], bx[3], bx[4], bx[6], c);
        standup_of(c, s4);
        float *g = geo + ((size_t)b * pre_max + i) * 12;
#pragma unroll
        for (int q = 0; q < 8; ++q) g[q] = c[q];
#pragma unroll
        for (int q = 0; q < 4; ++q) g[8 + q] = s4[q];
    }
}

// ------------------------------------------------------------------------------------------------
// pairwise suppression bitmask: grid (col_blocks, row_blocks, B), 256 threads = 64 rows x 4 col-quarters
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_iou_mask(const float *__restrict__ geo, const int *__restrict__ n_sorted, int pre_max, int words,
           int rotated, float thresh, float eps, int inclusive, unsigned long long *mask /*[B,pre_max,words]*/)
{
    const int b = blockIdx.z, rb = blockIdx.y, cb = blockIdx.x;
    const int n = n_sorted ? n_sorted[b] : pre_max;
    if (rb * 64 >= n || cb * 64 >= n || cb < rb) return;      // only the upper triangle of tiles is ever read
    __shared__ float s_col[64][12], s_row[64][12];
    __shared__ unsigned long long s_bits[64];
    __shared__ unsigned short s_queue[64 * 64];               // (row << 6 | col) of the pairs that need the polygon clip
    __shared__ int s_nq;
    const int tid = threadIdx.x;
    const float *gb = geo + (size_t)b * pre_max * 12;
    for (int i = tid; i < 64 * 12; i += 256) {
        int r = i / 12, q = i % 12;
        int j = cb * 64 + r, ii = rb * 64 + r;
        s_col[r][q] = (j < n) ? gb[(size_t)j * 12 + q] : 0.f;
        s_row[r][q] = (ii < n) ? gb[(size_t)ii * 12 + q] : 0.f;
    }
    if (tid < 64) s_bits[tid] = 0ull;
    if (tid == 0) s_nq = 0;
    __syncthreads();
    const int r = tid >> 2, quarter = tid & 3;
    const int i = rb * 64 + r;
    if (i < n) {
        unsigned long long bits = 0ull;
        for (int cc = 0; cc < 16; ++cc) {
            const int jl = quarter * 16 + cc;
            const int j = cb * 64 + jl;
            if (j >= n || j <= i) continue;
            if (rotated) {
                // cheap stand-up test here; the (divergent, ~500-instruction) polygon clip of the surviving pairs
                // is queued and spread evenly over the CTA below -- overlapping boxes cluster in a few rows, and a
                // warp would otherwise wait for its busiest lane
                const float *si = s_row[r] + 8, *sj = s_col[jl] + 8;
                const float iw = fminf(si[2], sj[2]) - fmaxf(si[0], sj[0]);
                const float ih = fminf(si[3], sj[3]) - fmaxf(si[1], sj[1]);
                if (iw > 0.f && ih > 0.f) s_queue[atomicAdd(&s_nq, 1)] = (unsigned short)((r << 6) | jl);
            } else if (suppress_aligned(s_row[r] + 8, s_col[jl] + 8, thresh, eps, inclusive != 0)) {
                bits |= 1ull << jl;
            }
        }
        if (bits) atomicOr(&s_bits[r], bits);
    }
    __syncthreads();
    if (rotated) {
        const int nq = s_nq;
        for (int q = tid; q < nq; q += 256) {
            const int rr = s_queue[q] >> 6, jl = s_queue[q] & 63;
            if (suppress_rotated(s_row[rr], s_row[rr] + 8, s_col[jl], s_col[jl] + 8, thresh))
                atomicOr(&s_bits[rr], 1ull << jl);
        }
        __syncthreads();
    }
    if (tid < 64 && rb * 64 + tid < n) mask[((size_t)b * pre_max + rb * 64 + tid) * words + cb] = s_bits[tid];
}

// ------------------------------------------------------------------------------------------------
// greedy reduce + epilogue: one CTA per frame
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_reduce_epilogue(const unsigned long long *__restrict__ mask, const int *__restrict__ n_sorted,
                  const int *__restrict__ sorted_slot, const float *__restrict__ cand_box,
                  const float *__restrict__ cand_score, const int *__restrict__ cand_label,
                  const int *__restrict__ cand_dir, int cand_cap, int code, int pre_max, int words,
                  int post_max, int use_dir, float dir_offset, float dir_limit_offset, int num_dir_bins,
                  int has_range, float r0, float r1, float r2, float r3, float r4, float r5, float *det,
                  int det_frame_stride, int *det_count)
{
    extern __shared__ __align__(16) unsigned char sm[];
    unsigned long long *s_mask = reinterpret_cast<unsigned long long *>(sm);  // [n][words]
    __shared__ int s_keep[1024];
    __shared__ int s_nkeep;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = n_sorted[b];
    const unsigned long long *mb = mask + (size_t)b * pre_max * words;
    // only words >= row/64 were written by k_iou_mask (upper triangle); lower words are never needed
    for (int i = tid; i < n * words; i += 256) {
        int r = i / words, w = i - r * words;
        s_mask[i] = (w >= (r >> 6) && w * 64 < n) ? mb[i] : 0ull;
    }
    __syncthreads();
    if (tid < 32) {
        const int lane = tid;
        unsigned long long removed = 0ull;  // lane holds word `lane` (pre_max <= 2048)
        // bits beyond n are "removed"
        {
            int lo = lane * 64;
            if (lo >= n) removed = ~0ull;
            else if (lo + 64 > n) removed = ~0ull << (n - lo);
        }
        int nk = 0;
        int cur = 0;
        while (nk < post_max) {
            // find the next not-removed index >= cur (warp-cooperative)
            unsigned long long avail = ~removed;
            int wcur = cur >> 6;
            if (lane < wcur) avail = 0ull;
            else if (lane == wcur) avail &= (~0ull << (cur & 63));
            unsigned ballot = __ballot_sync(0xffffffffu, avail != 0ull);
            if (ballot == 0u) break;
            int wl = __ffs(ballot) - 1;
            unsigned long long aw = __shfl_sync(0xffffffffu, avail, wl);
            int i = wl * 64 + (__ffsll((long long)aw) - 1);
            if (lane == 0) s_keep[nk] = i;
            ++nk;
            if (lane < words) removed |= s_mask[(size_t)i * words + lane];
            cur = i + 1;
        }
        if (lane == 0) s_nkeep = nk;
    }
    __syncthreads();
    const int nk = s_nkeep;
    // epilogue, one thread per kept box (loads in parallel; a serial loop of dependent global loads cost ~200 us):
    // pass 1 = range test -> s_keep[q] becomes the compacted output position (or -1); pass 2 = write.
    __shared__ int s_pos[1024];
    const int stride = code + 2;
    for (int q = tid; q < nk; q += 256) {
        int slot = sorted_slot[(size_t)b * pre_max + s_keep[q]];
        const float *bx = cand_box + ((size_t)b * cand_cap + slot) * code;
        bool ok = true;
        if (has_range) {
            float x = bx[0], y = bx[1], z = bx[2];
            ok = x >= r0 && y >= r1 && z >= r2 && x <= r3 && y <= r4 && z <= r5;
        }
        s_pos[q] = ok ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) {
        int out = 0;
        for (int q = 0; q < nk; ++q) {
            int f = s_pos[q];
            s_pos[q] = f ? out : -1;
            out += f;
        }
        det_count[b] = out;
        // record layout for the all-gather: the count rides in the record's last element
        if (det_frame_stride > post_max * stride) det[(size_t)b * det_frame_stride + det_frame_stride - 1] = (float)out;
    }
    __syncthreads();
    for (int q = tid; q < nk; q += 256) {
        const int pos = s_pos[q];
        if (pos < 0) continue;
        int slot = sorted_slot[(size_t)b * pre_max + s_keep[q]];
        size_t cs = (size_t)b * cand_cap + slot;
        const float *bx = cand_box + cs * code;
        float v[kMaxCode];
        for (int c = 0; c < code; ++c) v[c] = bx[c];
        if (use_dir) {
            // voxelnet.py:598-607: period = 2*pi/bins; r = limit_period(r - off, lim, period) + off + period*label
            float period = (float)(2.0 * 3.14159265358979323846 / (double)num_dir_bins);
            float val = __fsub_rn(v[6], dir_offset);
            float fl = floorf(__fadd_rn(__fdiv_rn(val, period), dir_limit_offset));
            float dir_rot = __fsub_rn(val, __fmul_rn(fl, period));
            v[6] = __fadd_rn(__fadd_rn(dir_rot, dir_offset), __fmul_rn(period, (float)cand_dir[cs]));
        }
        float *d = det + (size_t)b * det_frame_stride + (size_t)pos * stride;
        for (int c = 0; c < code; ++c) d[c] = v[c];
        d[code] = cand_score[cs];
        d[code + 1] = (float)cand_label[cs];
    }
}

struct NmsWorkspace {
    int *sorted_slot, *n_sorted;
    float *geo;
    unsigned long long *mask;
    int words;
};

size_t carve(NmsWorkspace *w, char *base, int batch, int pre_max)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += b2s_align(bytes); return base ? base + o : nullptr; };
    int words = (pre_max + 63) / 64;
    int *ss = (int *)take(sizeof(int) * (size_t)batch * pre_max);
    int *ns = (int *)take(sizeof(int) * (size_t)batch);
    float *geo = (float *)take(sizeof(float) * (size_t)batch * pre_max * 12);
    unsigned long long *mask = (unsigned long long *)take(sizeof(unsigned long long) * (size_t)batch * pre_max * words);
    if (w) { w->sorted_slot = ss; w->n_sorted = ns; w->geo = geo; w->mask = mask; w->words = words; }
    return off;
}

}  // namespace

static int decode_filter_launch(const float *box, const float *cls, const float *dir, HeadStrides hs,
                                const float *anchors, const uint8_t *anchors_mask, int batch, int a_loc, int H, int W,
                                int code, int ncls, int nbins, float score_thresh, float *cand_box, float *cand_score,
                                int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev, int cand_cap,
                                unsigned *status_dev, cudaStream_t stream)
{
    B2S_REQUIRE(code >= 7 && code <= kMaxCode && ncls >= 1 && batch >= 1 && a_loc >= 1 && cand_cap >= 1,
                "b2s_decode_filter: bad sizes");
    B2S_CUDA_OK(cudaMemsetAsync(cand_count_dev, 0, sizeof(int) * (size_t)batch, stream));
    long long total = (long long)batch * a_loc * H * W;
    k_decode_filter<<<b2s_cdiv(total, 256), 256, 0, stream>>>(box, cls, dir, hs, anchors, anchors_mask, batch, a_loc,
                                                             H, W, code, ncls, nbins, score_thresh, cand_box,
                                                             cand_score, cand_label, cand_dir, cand_anchor,
                                                             cand_count_dev, cand_cap, status_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_decode_filter(const float *box, const float *cls, const float *dir, const float *anchors,
                                 const uint8_t *anchors_mask, int batch, int a_loc, int H, int W, int code,
                                 int ncls, int nbins, float score_thresh, float *cand_box, float *cand_score,
                                 int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev,
                                 int cand_cap, unsigned *status_dev, void *stream_)
{
    // NCHW conv outputs: channel stride H*W, pixel stride 1
    HeadStrides hs;
    const long long HW = (long long)H * W;
    hs.box_b = (long long)a_loc * code * HW;
    hs.cls_b = (long long)a_loc * ncls * HW;
    hs.dir_b = (long long)a_loc * nbins * HW;
    hs.cs = (int)HW;
    hs.ps = 1;
    return decode_filter_launch(box, cls, dir, hs, anchors, anchors_mask, batch, a_loc, H, W, code, ncls, nbins,
                                score_thresh, cand_box, cand_score, cand_label, cand_dir, cand_anchor, cand_count_dev,
                                cand_cap, status_dev, (cudaStream_t)stream_);
}

extern "C" int b2s_decode_filter_strided(const float *box, const float *cls, const float *dir,
                                         long long box_batch_stride, long long cls_batch_stride,
                                         long long dir_batch_stride, int ch_stride, int pix_stride,
                                         const float *anchors, const uint8_t *anchors_mask, int batch, int a_loc,
                                         int H, int W, int code, int ncls, int nbins, float score_thresh,
                                         float *cand_box, float *cand_score, int *cand_label, int *cand_dir,
                                         int *cand_anchor, int *cand_count_dev, int cand_cap, unsigned *status_dev,
                                         void *stream_)
{
    HeadStrides hs;
    hs.box_b = box_batch_stride; hs.cls_b = cls_batch_stride; hs.dir_b = dir_batch_stride;
    hs.cs = ch_stride; hs.ps = pix_stride;
    return decode_filter_launch(box, cls, dir, hs, anchors, anchors_mask, batch, a_loc, H, W, code, ncls, nbins,
                                score_thresh, cand_box, cand_score, cand_label, cand_dir, cand_anchor, cand_count_dev,
                                cand_cap, status_dev, (cudaStream_t)stream_);
}

extern "C" int b2s_decode_filter_segments(const b2s_head_segment *segments, int num_segments, const float *anchors,
                                          const uint8_t *anchors_mask, int num_anchors, int batch, int code, int ncls,
                                          int nbins, float score_thresh, float *cand_box, float *cand_score,
                                          int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev,
                                          int cand_cap, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(segments != nullptr && num_segments >= 1 && num_segments <= B2S_MAX_HEAD_SEGMENTS,
                "b2s_decode_filter_segments: 1..4 segments");
    B2S_REQUIRE(code >= 7 && code <= kMaxCode && ncls >= 1 && batch >= 1 && num_anchors >= 1 && cand_cap >= 1,
                "b2s_decode_filter_segments: bad sizes");
    Segments sg;
    memset(&sg, 0, sizeof(sg));
    sg.n = num_segments;
    for (int i = 0; i < num_segments; ++i) {
        const b2s_head_segment &g = segments[i];
        B2S_REQUIRE(g.box != nullptr && g.cls != nullptr && g.a_loc >= 1 && g.H >= 1 && g.W >= 1 && g.anchor_base >= 0 &&
                        (long long)g.anchor_base + (long long)g.a_loc * g.H * g.W <= num_anchors,
                    "b2s_decode_filter_segments: segment %d lies outside [0, num_anchors) or has no box/cls tensor", i);
        for (int j = 0; j < i; ++j) {
            const b2s_head_segment &o = segments[j];
            const long long lo = g.anchor_base > o.anchor_base ? g.anchor_base : o.anchor_base;
            const long long e1 = (long long)g.anchor_base + (long long)g.a_loc * g.H * g.W;
            const long long e2 = (long long)o.anchor_base + (long long)o.a_loc * o.H * o.W;
            B2S_REQUIRE(lo >= (e1 < e2 ? e1 : e2), "b2s_decode_filter_segments: segments %d and %d overlap", j, i);
        }
        sg.box[i] = g.box; sg.cls[i] = g.cls; sg.dir[i] = g.dir;
        sg.hs[i].box_b = g.box_batch_stride; sg.hs[i].cls_b = g.cls_batch_stride; sg.hs[i].dir_b = g.dir_batch_stride;
        sg.hs[i].cs = g.ch_stride; sg.hs[i].ps = g.pix_stride;
        sg.a_loc[i] = g.a_loc; sg.H[i] = g.H; sg.W[i] = g.W; sg.base[i] = g.anchor_base;
    }
    B2S_CUDA_OK(cudaMemsetAsync(cand_count_dev, 0, sizeof(int) * (size_t)batch, stream));
    long long total = (long long)batch * num_anchors;
    k_decode_filter_segments<<<b2s_cdiv(total, 256), 256, 0, stream>>>(
        sg, anchors, anchors_mask, batch, num_anchors, code, ncls, nbins, score_thresh, cand_box, cand_score, cand_label,
        cand_dir, cand_anchor, cand_count_dev, cand_cap, status_dev);
    B2S_LAUNCH_OK();
    return 0;
}

// multi-class NMS branch: per-(class, frame) candidate lists (class-major virtual frames, see k_decode_filter_mc).
// Head tensors by strides like b2s_decode_filter_strided.  class_lo/class_hi: a_loc index range per class (host
// [ncls]; NULL = class-agnostic: every anchor competes in every class); score_thresh host [ncls].
extern "C" int b2s_decode_filter_multiclass(const float *box, const float *cls, const float *dir,
                                            long long box_batch_stride, long long cls_batch_stride,
                                            long long dir_batch_stride, int ch_stride, int pix_stride,
                                            const float *anchors, int batch, int a_loc, int H, int W, int code, int ncls,
                                            int nbins, const int *class_lo, const int *class_hi,
                                            const float *score_thresh, float *cand_box, float *cand_score,
                                            int *cand_label, int *cand_dir, int *cand_anchor, int *cand_count_dev,
                                            int cand_cap, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(code >= 7 && code <= kMaxCode && ncls >= 1 && ncls <= 16 && batch >= 1 && a_loc >= 1 && cand_cap >= 1,
                "b2s_decode_filter_multiclass: bad sizes (ncls <= 16)");
    B2S_REQUIRE(score_thresh != nullptr && ((class_lo == nullptr) == (class_hi == nullptr)),
                "b2s_decode_filter_multiclass: score_thresh required; class_lo/class_hi both or neither");
    HeadStrides hs;
    hs.box_b = box_batch_stride; hs.cls_b = cls_batch_stride; hs.dir_b = dir_batch_stride;
    hs.cs = ch_stride; hs.ps = pix_stride;
    ClassRanges cr;
    for (int c = 0; c < 16; ++c) {
        cr.lo[c] = (c < ncls && class_lo) ? class_lo[c] : 0;
        cr.hi[c] = (c < ncls && class_hi) ? class_hi[c] : a_loc;
        cr.thresh[c] = c < ncls ? score_thresh[c] : 2.f;
    }
    B2S_CUDA_OK(cudaMemsetAsync(cand_count_dev, 0, sizeof(int) * (size_t)batch * ncls, stream));
    long long total = (long long)batch * a_loc * H * W;
    k_decode_filter_mc<<<b2s_cdiv(total, 256), 256, 0, stream>>>(box, cls, dir, hs, anchors, batch, a_loc, H, W, code, ncls,
                                                                nbins, cr, cand_box, cand_score, cand_label, cand_dir,
                                                                cand_anchor, cand_count_dev, cand_cap, status_dev);
    B2S_LAUNCH_OK();
    return 0;
}

// det_mc [ncls*batch, post_max, code+2] + count_mc [ncls*batch] (class-major, the b2s_nms outputs of the virtual
// frames) -> per-frame records in class order; det / det_frame_stride / det_count_dev as in b2s_nms with
// ncls*post_max rows per frame.
extern "C" int b2s_concat_class_detections(const float *det_mc, const int *count_mc, int batch, int ncls, int post_max,
                                           int code, float *det, int det_frame_stride, int *det_count_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && ncls >= 1 && ncls <= 16 && post_max >= 1, "b2s_concat_class_detections: bad sizes");
    const int S = code + 2;
    if (det_frame_stride == 0) det_frame_stride = ncls * post_max * S;
    B2S_REQUIRE(det_frame_stride >= ncls * post_max * S, "b2s_concat_class_detections: det_frame_stride too small");
    k_concat_classes<<<batch, 256, 0, stream>>>(det_mc, count_mc, batch, ncls, post_max, S, det, det_frame_stride,
                                                det_count_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" size_t b2s_nms_workspace_bytes(int batch, int cand_cap, int pre_max)
{
    (void)cand_cap;
    return carve(nullptr, nullptr, batch, pre_max);
}

static int launch_mask_reduce(const NmsWorkspace &w, int batch, int pre_max, int rotated, float iou_thresh,
                              cudaStream_t stream)
{
    int nb = (pre_max + 63) / 64;
    dim3 grid(nb, nb, batch);
    k_iou_mask<<<grid, 256, 0, stream>>>(w.geo, w.n_sorted, pre_max, w.words, rotated, iou_thresh, 1.f, 0, w.mask);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_nms(const float *cand_box, const float *cand_score, const int *cand_label,
                       const int *cand_dir, const int *cand_anchor, const int *cand_count_dev, int batch,
                       int cand_cap, int code, int rotated, int pre_max, int post_max, float iou_thresh,
                       int use_dir, float dir_offset, float dir_limit_offset, int num_dir_bins,
                       const float *range_host, float *det, int det_frame_stride, int *det_count_dev,
                       void *workspace, size_t workspace_bytes, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(pre_max >= 1 && pre_max <= 2048, "b2s_nms: pre_max must be 1..2048");
    B2S_REQUIRE(post_max >= 1 && post_max <= 1024, "b2s_nms: post_max must be 1..1024");
    B2S_REQUIRE(code >= 7 && code <= kMaxCode, "b2s_nms: bad code size");
    if (det_frame_stride == 0) det_frame_stride = post_max * (code + 2);
    B2S_REQUIRE(det_frame_stride >= post_max * (code + 2), "b2s_nms: det_frame_stride smaller than a frame's rows");
    NmsWorkspace w;
    size_t need = carve(&w, (char *)workspace, batch, pre_max);
    B2S_REQUIRE(workspace_bytes >= need, "b2s_nms: workspace too small (%zu < %zu)", workspace_bytes, need);
    static bool attr_set[64] = {false};      // per device: the attribute belongs to the current device
    int cur_dev = 0;
    B2S_CUDA_OK(cudaGetDevice(&cur_dev));
    cur_dev &= 63;
    size_t smem_sel = (size_t)kSortCap * (sizeof(unsigned long long) + sizeof(int));
    size_t smem_red = sizeof(unsigned long long) * (size_t)pre_max * w.words;
    if (!attr_set[cur_dev]) {
        B2S_CUDA_OK(cudaFuncSetAttribute(k_select_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
        B2S_CUDA_OK(cudaFuncSetAttribute(k_reduce_epilogue, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_set[cur_dev] = true;
    }
    B2S_REQUIRE(smem_red <= 200 * 1024, "b2s_nms: pre_max too large for the shared-memory reduce");
    k_select_sort<<<batch, kSelThreads, smem_sel, stream>>>(cand_box, cand_score, cand_anchor, cand_count_dev,
                                                           cand_cap, code, pre_max, w.sorted_slot, w.geo,
                                                           w.n_sorted);
    B2S_LAUNCH_OK();
    if (launch_mask_reduce(w, batch, pre_max, rotated, iou_thresh, stream) != 0) return -1;
    float r[6] = {0, 0, 0, 0, 0, 0};
    if (range_host) for (int i = 0; i < 6; ++i) r[i] = range_host[i];
    k_reduce_epilogue<<<batch, 256, smem_red, stream>>>(w.mask, w.n_sorted, w.sorted_slot, cand_box, cand_score,
                                                       cand_label, cand_dir, cand_cap, code, pre_max, w.words,
                                                       post_max, use_dir, dir_offset, dir_limit_offset,
                                                       num_dir_bins, range_host != nullptr, r[0], r[1], r[2],
                                                       r[3], r[4], r[5], det, det_frame_stride, det_count_dev);
    B2S_LAUNCH_OK();
    return 0;
}

// ------------------------------------------------------------------------------------------------
// numpy-facing wrappers (host arrays, internal copies + sync, like upstream's non_max_suppression)
// ------------------------------------------------------------------------------------------------
namespace {

__global__ void k_geo_from_dets(const float *__restrict__ dets, int n, float *geo)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float *g = geo + (size_t)i * 12;
    for (int q = 0; q < 8; ++q) g[q] = 0.f;
    for (int q = 0; q < 4; ++q) g[8 + q] = dets[(size_t)i * 5 + q];
}

// corners given by the caller; stand-up gate given as a matrix -> fold the gate into the mask kernel by
// recomputing stand-up boxes from the corners (identical to corner_to_standup_nd + iou_jit(eps=0) > 0).
__global__ void k_geo_from_corners(const float *__restrict__ corners, const int *__restrict__ order, int n,
                                   float *geo)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *c = corners + (size_t)order[i] * 8;
    float *g = geo + (size_t)i * 12;
    float cc[8], s4[4];
    for (int q = 0; q < 8; ++q) { cc[q] = c[q]; g[q] = c[q]; }
    standup_of(cc, s4);
    for (int q = 0; q < 4; ++q) g[8 + q] = s4[q];
}

__global__ void k_reduce_simple(const unsigned long long *__restrict__ mask, int n, int words, int *keep,
                                int *nkeep)
{
    // single warp, global-memory rows (compat path; n <= 2048*... any n: words may exceed 32 -> loop)
    extern __shared__ unsigned long long s_removed[];
    for (int w = threadIdx.x; w < words; w += blockDim.x) s_removed[w] = 0ull;
    __syncthreads();
    if (threadIdx.x >= 32) return;
    int nk = 0;
    for (int i = 0; i < n; ++i) {
        bool rem = (s_removed[i >> 6] >> (i & 63)) & 1ull;
        if (rem) continue;
        if (threadIdx.x == 0) keep[nk] = i;
        ++nk;
        for (int w = (i >> 6) + threadIdx.x; w < words; w += 32) s_removed[w] |= mask[(size_t)i * words + w];
        __syncwarp();
    }
    if (threadIdx.x == 0) *nkeep = nk;
}

// RAII for the numpy-facing wrappers: temporaries are freed and the caller's current device is restored on EVERY
// exit path (upstream's *_cpu functions never touch CUDA state, so ours must not leave a different device current)
struct DeviceScope {
    int prev = -1;
    bool ok = true;
    explicit DeviceScope(int device_id)
    {
        if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; ok = false; return; }
        if (device_id >= 0 && device_id != prev) ok = cudaSetDevice(device_id) == cudaSuccess;
    }
    ~DeviceScope()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};
struct DevBuf {
    void *p = nullptr;
    cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
    ~DevBuf()
    {
        if (p) cudaFree(p);
    }
    template <typename T> T *as() { return reinterpret_cast<T *>(p); }
};

int host_nms_common(float *d_geo, int n, int rotated, float thresh, float eps, int inclusive, int *keep_out_host,
                    cudaStream_t stream)
{
    int words = (n + 63) / 64;
    DevBuf mask, keep, nkeep;
    B2S_CUDA_OK(mask.alloc(sizeof(unsigned long long) * (size_t)n * words));
    B2S_CUDA_OK(keep.alloc(sizeof(int) * (size_t)n));
    B2S_CUDA_OK(nkeep.alloc(sizeof(int)));
    B2S_CUDA_OK(cudaMemsetAsync(mask.p, 0, sizeof(unsigned long long) * (size_t)n * words, stream));
    dim3 grid(words, words, 1);
    k_iou_mask<<<grid, 256, 0, stream>>>(d_geo, nullptr, n, words, rotated, thresh, eps, inclusive,
                                         mask.as<unsigned long long>());
    B2S_LAUNCH_OK();
    k_reduce_simple<<<1, 32, sizeof(unsigned long long) * words, stream>>>(mask.as<unsigned long long>(), n, words,
                                                                           keep.as<int>(), nkeep.as<int>());
    B2S_LAUNCH_OK();
    int nk = 0;
    B2S_CUDA_OK(cudaMemcpyAsync(&nk, nkeep.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
    B2S_CUDA_OK(cudaStreamSynchronize(stream));
    if (nk > 0) B2S_CUDA_OK(cudaMemcpy(keep_out_host, keep.p, sizeof(int) * (size_t)nk, cudaMemcpyDeviceToHost));
    return nk;
}

// rotated overlap of every (box n, query k) pair: one thread per pair (N x K is small: eval / target assignment)
//   criterion -1: IoU, 0: inter/area(box), 1: inter/area(query), 2: intersection area
//   (second/core/non_max_suppression/nms_gpu.py:553-566 devRotateIoUEval)
__device__ __forceinline__ float overlap_of(float inter, float area_b, float area_q, int criterion)
{
    if (criterion == -1) return inter / (area_b + area_q - inter);
    if (criterion == 0) return inter / area_b;
    if (criterion == 1) return inter / area_q;
    return inter;
}

__global__ void k_rbbox_pairs(const float *__restrict__ corners, const float *__restrict__ qcorners,
                              const float *__restrict__ standup_iou, int N, int K, float standup_thresh, int criterion,
                              float *__restrict__ out)
{
    const long long total = (long long)N * K;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(g / K), k = (int)(g % K);
        float r = 0.f;
        bool gate;
        float a[8], b[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { a[i] = corners[(size_t)n * 8 + i]; b[i] = qcorners[(size_t)k * 8 + i]; }
        if (standup_iou) {
            gate = standup_iou[g] > standup_thresh;
        } else {                      // gate = stand-up boxes overlap (iou_jit(eps=0) > 0)
            float sa[4], sb[4];
            standup_of(a, sa);
            standup_of(b, sb);
            gate = fminf(sa[2], sb[2]) - fmaxf(sa[0], sb[0]) > 0.f && fminf(sa[3], sb[3]) - fmaxf(sa[1], sb[1]) > 0.f;
        }
        if (gate) {
            float area_a, area_b;
            const float inter = quad_intersection(a, b, &area_a, &area_b);
            r = overlap_of(inter, area_a, area_b, criterion);
        }
        out[g] = r;
    }
}

__global__ void k_corners_from_rboxes(const float *__restrict__ boxes /*[n,5] x,y,w,l,r*/, int n, float *corners)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *b = boxes + (size_t)i * 5;
    float c[8];
    bev_corners(b[0], b[1], b[2], b[3], b[4], c);
#pragma unroll
    for (int q = 0; q < 8; ++q) corners[(size_t)i * 8 + q] = c[q];
}

}  // namespace

extern "C" int b2s_nms_aligned_host(const float *sorted_dets, int n, float thresh, float eps, int inclusive,
                                    int *keep_out, int device_id)
{
    if (n <= 0) return 0;
    DeviceScope scope(device_id);
    B2S_REQUIRE(scope.ok, "b2s_nms_aligned_host: cannot select device %d", device_id);
    DevBuf dets, geo;
    B2S_CUDA_OK(dets.alloc(sizeof(float) * (size_t)n * 5));
    B2S_CUDA_OK(geo.alloc(sizeof(float) * (size_t)n * 12));
    B2S_CUDA_OK(cudaMemcpy(dets.p, sorted_dets, sizeof(float) * (size_t)n * 5, cudaMemcpyHostToDevice));
    k_geo_from_dets<<<b2s_cdiv(n, 256), 256>>>(dets.as<float>(), n, geo.as<float>());
    B2S_LAUNCH_OK();
    return host_nms_common(geo.as<float>(), n, 0, thresh, eps, inclusive, keep_out, 0);
}

extern "C" int b2s_nms_rotated_host(const float *corners, const int *order, const float *standup_iou, int n,
                                    float thresh, int *keep_out, int device_id)
{
    (void)standup_iou;  // gate recomputed on the device from the corners (same predicate)
    if (n <= 0) return 0;
    DeviceScope scope(device_id);
    B2S_REQUIRE(scope.ok, "b2s_nms_rotated_host: cannot select device %d", device_id);
    DevBuf c, geo, ord;
    B2S_CUDA_OK(c.alloc(sizeof(float) * (size_t)n * 8));
    B2S_CUDA_OK(geo.alloc(sizeof(float) * (size_t)n * 12));
    B2S_CUDA_OK(ord.alloc(sizeof(int) * (size_t)n));
    B2S_CUDA_OK(cudaMemcpy(c.p, corners, sizeof(float) * (size_t)n * 8, cudaMemcpyHostToDevice));
    B2S_CUDA_OK(cudaMemcpy(ord.p, order, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice));
    k_geo_from_corners<<<b2s_cdiv(n, 256), 256>>>(c.as<float>(), ord.as<int>(), n, geo.as<float>());
    B2S_LAUNCH_OK();
    int *keep_sorted = (int *)malloc(sizeof(int) * (size_t)n);
    if (!keep_sorted) { b2s_set_error("b2s_nms_rotated_host: out of host memory"); return -1; }
    int nk = host_nms_common(geo.as<float>(), n, 1, thresh, 0.f, 1, keep_sorted, 0);
    for (int i = 0; i < nk; ++i) keep_out[i] = order[keep_sorted[i]];  // positions in `order` -> box ids
    free(keep_sorted);
    return nk;
}

// Device-resident rotated overlap matrix (the rotate_iou_gpu_eval replacement, nms_gpu.py:569-607): boxes [N,5],
// query_boxes [K,5] as (x, y, w, l, r); out [N,K].  workspace: (N + K) * 8 floats.
extern "C" int b2s_rotate_iou_eval(const float *boxes, int N, const float *query_boxes, int K, int criterion, float *out,
                                   float *workspace, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(N >= 0 && K >= 0 && criterion >= -1 && criterion <= 2, "b2s_rotate_iou_eval: bad arguments");
    if (N == 0 || K == 0) return 0;
    float *c = workspace, *qc = workspace + (size_t)N * 8;
    k_corners_from_rboxes<<<b2s_cdiv(N, 256), 256, 0, stream>>>(boxes, N, c);
    B2S_LAUNCH_OK();
    k_corners_from_rboxes<<<b2s_cdiv(K, 256), 256, 0, stream>>>(query_boxes, K, qc);
    B2S_LAUNCH_OK();
    long long total = (long long)N * K;
    int blocks = b2s_cdiv(total, 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    k_rbbox_pairs<<<blocks, 256, 0, stream>>>(c, qc, nullptr, N, K, 0.f, criterion, out);
    B2S_LAUNCH_OK();
    return 0;
}

// spconv.utils.rbbox_iou (criterion -1) / rbbox_intersection (criterion 2) with the numpy-facing contract: HOST
// arrays in and out (second/core/box_np_ops.py:10-34).
extern "C" int b2s_rbbox_overlap_host(const float *corners, const float *qcorners, const float *standup_iou, int N, int K,
                                      float standup_thresh, int criterion, float *out, int device_id)
{
    if (N <= 0 || K <= 0) return 0;
    B2S_REQUIRE(criterion >= -1 && criterion <= 2 && standup_iou != nullptr, "b2s_rbbox_overlap_host: bad arguments");
    DeviceScope scope(device_id);
    B2S_REQUIRE(scope.ok, "b2s_rbbox_overlap_host: cannot select device %d", device_id);
    DevBuf c, qc, si, o;
    B2S_CUDA_OK(c.alloc(sizeof(float) * (size_t)N * 8));
    B2S_CUDA_OK(qc.alloc(sizeof(float) * (size_t)K * 8));
    B2S_CUDA_OK(si.alloc(sizeof(float) * (size_t)N * K));
    B2S_CUDA_OK(o.alloc(sizeof(float) * (size_t)N * K));
    B2S_CUDA_OK(cudaMemcpy(c.p, corners, sizeof(float) * (size_t)N * 8, cudaMemcpyHostToDevice));
    B2S_CUDA_OK(cudaMemcpy(qc.p, qcorners, sizeof(float) * (size_t)K * 8, cudaMemcpyHostToDevice));
    B2S_CUDA_OK(cudaMemcpy(si.p, standup_iou, sizeof(float) * (size_t)N * K, cudaMemcpyHostToDevice));
    long long total = (long long)N * K;
    int blocks = b2s_cdiv(total, 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    k_rbbox_pairs<<<blocks, 256>>>(c.as<float>(), qc.as<float>(), si.as<float>(), N, K, standup_thresh, criterion,
                                   o.as<float>());
    B2S_LAUNCH_OK();
    B2S_CUDA_OK(cudaMemcpy(out, o.p, sizeof(float) * (size_t)N * K, cudaMemcpyDeviceToHost));
    return 0;
}
