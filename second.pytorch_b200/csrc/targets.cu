// targets.cu -- training targets of TargetAssigner.assign (second/core/target_assigner.py:38-167) through
// create_target_np (second/core/target_ops.py:29-229) with positive_fraction None, for a batch of frames.
//
// A segment is a range of anchors with one similarity (one class's anchors in per-class mode, every anchor in
// assign_all); frame b's ground truths of segment s occupy sorted slots [seg_off[b][s], seg_off[b][s+1]).
//   k_ta_gt_prep<T>   one block per frame: stable partition of the frame's GTs into segments (perm), each GT's
//                     rbbox2d_to_near_bbox (box_np_ops.py:286-298) in the GT's own dtype T, per-GT max keys zeroed
//   k_ta_pass<T, 0>   one thread per (frame, anchor): the similarity to every GT of its segment, staged through shared
//                     memory kChunk GTs at a time; per-GT maxima over unpruned anchors as atomicMax on ordered uint32
//                     keys (a warp max first, then shared, then global)
//   k_ta_pass<T, 1>   the same similarities again (same bits), the anchor's max / first argmax and the forced flag
//                     (similarity == some GT's max), then label, importance and GroundBox3dCoder.encode.
// The similarities follow numba's typing of iou_jit(eps=0.0) (box_np_ops.py:697-725) and distance_similarity
// (:950-973): float32 anchors, GT of dtype T, promoted to float64 where eps / dist_norm enter, stored as float32.  Every
// arithmetic step is an explicit round-to-nearest intrinsic, so --fmad=true cannot contract it; labels depend on
// equality ties and need the reference's bits.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 128;
constexpr int kMaxSegments = 64;
constexpr int kSimIou = 0;
constexpr int kSimDistance = 1;

template <typename T> struct Ar;
template <> struct Ar<float> {
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
    static __device__ __forceinline__ float lo(float a, float b) { return fminf(a, b); }
    static __device__ __forceinline__ float hi(float a, float b) { return fmaxf(a, b); }
    static __device__ __forceinline__ float log_(float a) { return logf(a); }
    static __device__ __forceinline__ float cos_(float a) { return cosf(a); }
    static __device__ __forceinline__ float sin_(float a) { return sinf(a); }
    static __device__ __forceinline__ float to_f32(float a) { return a; }
    static constexpr float kPi = (float)M_PI;
    static constexpr float kQuarterPi = (float)(M_PI / 4);   // numpy compares float32 with a weak Python float in float32
};
template <> struct Ar<double> {
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
    static __device__ __forceinline__ double lo(double a, double b) { return fmin(a, b); }
    static __device__ __forceinline__ double hi(double a, double b) { return fmax(a, b); }
    static __device__ __forceinline__ double log_(double a) { return log(a); }
    static __device__ __forceinline__ double cos_(double a) { return cos(a); }
    static __device__ __forceinline__ double sin_(double a) { return sin(a); }
    static __device__ __forceinline__ float to_f32(double a) { return __double2float_rn(a); }
    static constexpr double kPi = M_PI;
    static constexpr double kQuarterPi = M_PI / 4;
};

// order-preserving float -> uint32 key; -0 is canonicalised to +0 (numpy's == treats them as equal); key 0 stays free
// and means "no unpruned anchor"
__device__ __forceinline__ uint32_t f2key(float f)
{
    const uint32_t u = __float_as_uint(f == 0.f ? 0.f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key2f(uint32_t k)
{
    if (k == 0) return __int_as_float(0x7fc00000);           // NaN: equal to nothing, so forces nothing
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct Params {
    const float *anchors;           // [A, ndim]
    const float4 *anchor_sim;       // [A]: near bbox (IoU segments) or (x, y, 0, 0) (distance segments)
    const float *matched, *unmatched;
    int A, ndim;
    const int4 *seg_info;           // [S]: (anchor_begin, anchor_end, kind, 0)
    const double *seg_param;        // [S]: distance_norm
    int S;
    const int4 *blocks;             // [NB]: (segment, anchor_begin, anchor_end, 0), at most kThreads anchors
    const void *gt;                 // [G, ndim] of T
    const int *gt_off;              // [B+1]
    const int *gt_seg, *gt_class;   // [G]
    const float *gt_imp;            // [G] or null
    int G;
    const uint8_t *mask;            // [B, A] or null
    int code, linear_dim, vec_encode;
    int *perm;                      // [G] sorted slot -> packed GT index
    int *seg_off;                   // [B, S+1] sorted slots
    void *gt_nb;                    // [G, 4] of T, sorted slots
    uint32_t *gt_key;               // [G] sorted slots
    int *labels;
    float *targets, *importance;
    int *gt_id;                     // optional [B, A]
    float *overlap;                 // optional [B, A]
    unsigned *status;
};

// rbbox2d_to_near_bbox of one box (x, y, z, w, l, h, r) with limit_period(r, 0.5, pi) and center_to_minmax_2d
template <typename T>
__device__ __forceinline__ void near_bbox(const T *box, T out[4])
{
    using M = Ar<T>;
    const T r = box[6];
    const T q = floor(M::add(M::div(r, M::kPi), T(0.5)));
    const T rp = fabs(M::sub(r, M::mul(q, M::kPi)));
    const bool swap = rp > M::kQuarterPi;
    const T dx = swap ? box[4] : box[3], dy = swap ? box[3] : box[4];
    const T hx = M::mul(dx, T(0.5)), hy = M::mul(dy, T(0.5));        // dims / 2, exact
    out[0] = M::sub(box[0], hx);
    out[1] = M::sub(box[1], hy);
    out[2] = M::add(box[0], hx);
    out[3] = M::add(box[1], hy);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_ta_gt_prep(Params p)
{
    __shared__ int s_cursor[kMaxSegments + 1];
    __shared__ int s_warp[kThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    int f0 = p.gt_off[b], f1 = p.gt_off[b + 1];
    if (f0 < 0 || f1 < f0 || f1 > p.G) {
        if (tid == 0) atomicOr(p.status, B2S_STATUS_BAD_INPUT);
        f0 = f1 = 0;                                               // the frame is treated as having no GT
    }
    for (int s = tid; s <= p.S; s += kThreads) s_cursor[s] = 0;
    __syncthreads();
    for (int g = f0 + tid; g < f1; g += kThreads) {
        const int s = p.gt_seg[g];
        if ((unsigned)s < (unsigned)p.S) atomicAdd(&s_cursor[s], 1);
    }
    __syncthreads();
    if (tid == 0) {
        int acc = f0;
        for (int s = 0; s < p.S; ++s) {
            const int c = s_cursor[s];
            s_cursor[s] = acc;
            p.seg_off[b * (p.S + 1) + s] = acc;
            acc += c;
        }
        s_cursor[p.S] = acc;
        p.seg_off[b * (p.S + 1) + p.S] = acc;
    }
    __syncthreads();
    // stable placement: within a chunk, a GT's rank among the chunk's GTs of its segment comes from a ballot
    for (int c0 = f0; c0 < f1; c0 += kThreads) {
        const int g = c0 + tid;
        const int sg = g < f1 ? p.gt_seg[g] : -1;
        for (int s = 0; s < p.S; ++s) {
            const unsigned bal = __ballot_sync(0xffffffffu, sg == s);
            if (lane == 0) s_warp[wid] = __popc(bal);
            __syncthreads();
            if (sg == s) {
                int pos = s_cursor[s] + __popc(bal & ((1u << lane) - 1u));
                for (int w = 0; w < wid; ++w) pos += s_warp[w];
                p.perm[pos] = g;
            }
            __syncthreads();
            if (tid == 0) {
                int t = 0;
                for (int w = 0; w < kThreads / 32; ++w) t += s_warp[w];
                s_cursor[s] += t;
            }
            __syncthreads();
        }
    }
    const int end = s_cursor[p.S];                                 // == seg_off[b][S] after the placement
    const T *gt = static_cast<const T *>(p.gt);
    T *nb = static_cast<T *>(p.gt_nb);
    for (int j = f0 + tid; j < end; j += kThreads) {
        const int g = p.perm[j];
        const T *box = gt + (size_t)g * p.ndim;
        T o[4];
        if (__ldg(&p.seg_info[p.gt_seg[g]].z) == kSimDistance) {
            o[0] = box[0]; o[1] = box[1]; o[2] = T(0); o[3] = T(0);
        } else {
            near_bbox<T>(box, o);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) nb[(size_t)j * 4 + k] = o[k];
        p.gt_key[j] = 0u;
    }
}

// similarity of an anchor (float32) with a staged GT (T); a_area = the anchor's (x1-x0)*(y1-y0) in float64
template <typename T>
__device__ __forceinline__ float similarity(int kind, double dn, const float4 av, double a_area, const T q[4],
                                            double q_area)
{
    using M = Ar<T>;
    if (kind == kSimIou) {
        const double iw = (double)M::sub(M::lo(T(av.z), q[2]), M::hi(T(av.x), q[0]));
        if (iw > 0) {
            const double ih = (double)M::sub(M::lo(T(av.w), q[3]), M::hi(T(av.y), q[1]));
            if (ih > 0) {
                const double inter = __dmul_rn(iw, ih);
                const double ua = __dsub_rn(__dadd_rn(a_area, q_area), inter);
                return __double2float_rn(__ddiv_rn(inter, ua));
            }
        }
        return 0.f;
    }
    const T dx = M::sub(T(av.x), q[0]);
    if ((double)fabs(dx) <= dn) {
        const T dy = M::sub(T(av.y), q[1]);
        if ((double)fabs(dy) <= dn) {
            const T dist = M::add(M::mul(dx, dx), M::mul(dy, dy));
            const double dnorm = fmin(__ddiv_rn((double)dist, dn), dn);
            return __double2float_rn(__dsub_rn(1.0, dnorm));
        }
    }
    return 0.f;
}

// GroundBox3dCoder.encode = second_box_encode(boxes, anchors, vec_encode, linear_dim) (box_np_ops.py:36-83), each
// expression in numpy's promoted dtype of its operands, stored through float32
template <typename T>
__device__ __forceinline__ void encode(const Params &p, const T *g, const float *a, float *out)
{
    using M = Ar<T>;
    const float diag = __fsqrt_rn(__fadd_rn(__fmul_rn(a[4], a[4]), __fmul_rn(a[3], a[3])));
    out[0] = M::to_f32(M::div(M::sub(g[0], T(a[0])), T(diag)));
    out[1] = M::to_f32(M::div(M::sub(g[1], T(a[1])), T(diag)));
    out[2] = M::to_f32(M::div(M::sub(g[2], T(a[2])), T(a[5])));
#pragma unroll
    for (int k = 3; k < 6; ++k) {                                   // wt, lt, ht
        const T r = M::div(g[k], T(a[k]));
        out[k] = M::to_f32(p.linear_dim ? M::sub(r, T(1)) : M::log_(r));
    }
    int o = 6;
    if (p.vec_encode) {
        out[o++] = M::to_f32(M::sub(M::cos_(g[6]), T(cosf(a[6]))));
        out[o++] = M::to_f32(M::sub(M::sin_(g[6]), T(sinf(a[6]))));
    } else {
        out[o++] = M::to_f32(M::sub(g[6], T(a[6])));
    }
    for (int k = 7; k < p.ndim; ++k) out[o++] = M::to_f32(M::sub(g[k], T(a[k])));
}

template <typename T, bool kFinal>
__global__ void __launch_bounds__(kThreads) k_ta_pass(Params p)
{
    __shared__ T s_nb[kChunk][4];
    __shared__ double s_area[kChunk];
    __shared__ uint32_t s_key[kChunk];
    __shared__ float s_max[kChunk];
    const int4 blk = __ldg(&p.blocks[blockIdx.x]);
    const int b = blockIdx.y, seg = blk.x, lane = threadIdx.x & 31;
    const int a = blk.y + threadIdx.x;
    const bool in = a < blk.z;
    const size_t o = (size_t)b * p.A + a;
    const bool active = in && (p.mask == nullptr || p.mask[o] != 0);
    const int g0 = p.seg_off[b * (p.S + 1) + seg], g1 = p.seg_off[b * (p.S + 1) + seg + 1];
    const int kind = __ldg(&p.seg_info[seg].z);
    const double dn = __ldg(&p.seg_param[seg]);
    const float4 av = in ? __ldg(&p.anchor_sim[a]) : make_float4(0.f, 0.f, 0.f, 0.f);
    const double a_area = __dmul_rn((double)__fsub_rn(av.z, av.x), (double)__fsub_rn(av.w, av.y));
    const bool warp_active = __any_sync(0xffffffffu, active);
    const T *nb = static_cast<const T *>(p.gt_nb);
    float best = -INFINITY;
    int arg = 0;
    bool forced = false;
    for (int c0 = g0; c0 < g1; c0 += kChunk) {
        const int n = min(kChunk, g1 - c0);
        __syncthreads();                                           // the previous chunk is consumed
        for (int j = threadIdx.x; j < n; j += kThreads) {
            T q[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) q[k] = nb[(size_t)(c0 + j) * 4 + k];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_nb[j][k] = q[k];
            // box_area of iou_jit: (q2 - q0 + eps) * (q3 - q1 + eps), the differences in T, the product in float64
            s_area[j] = __dmul_rn((double)Ar<T>::sub(q[2], q[0]), (double)Ar<T>::sub(q[3], q[1]));
            if (kFinal) {
                const float m = key2f(p.gt_key[c0 + j]);
                s_max[j] = m == 0.f ? -1.f : m;                     // gt_to_anchor_max == 0 -> -1
            } else {
                s_key[j] = 0u;
            }
        }
        __syncthreads();
        if (warp_active) {
            for (int j = 0; j < n; ++j) {
                T q[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) q[k] = s_nb[j][k];
                const float s = active ? similarity<T>(kind, dn, av, a_area, q, s_area[j]) : 0.f;
                if (kFinal) {
                    if (active) {
                        if (s > best) { best = s; arg = c0 + j - g0; }   // first index on ties
                        forced |= (s == s_max[j]);
                    }
                } else {
                    const uint32_t k = __reduce_max_sync(0xffffffffu, active ? f2key(s) : 0u);
                    if (lane == 0 && k != 0u) atomicMax(&s_key[j], k);
                }
            }
        }
        if (!kFinal) {
            __syncthreads();
            for (int j = threadIdx.x; j < n; j += kThreads) {
                const uint32_t k = s_key[j];
                // keys only grow: a key at or below the value already stored cannot change it
                if (k > *(volatile uint32_t *)&p.gt_key[c0 + j]) atomicMax(&p.gt_key[c0 + j], k);
            }
        }
    }
    if (!kFinal || !in) return;

    float *tgt = p.targets + o * p.code;
    int label = -1, gid = -1;
    float imp = 0.f;
    bool fg = false;
    if (active) {
        if (g1 == g0) {
            label = 0;                                             // no GT in the segment: every anchor is background
            imp = 1.f;
        } else {
            const int g = p.perm[g0 + arg];
            const int cls = p.gt_class[g];
            const bool pos = best >= p.matched[a];
            // write order of target_ops.py:130-173: forced, then >= matched, then the bg overwrite, forced again
            label = forced ? cls : (best < p.unmatched[a] ? 0 : (pos ? cls : -1));
            // importance[pos_inds] = gt_importance[gt_inds]: the class-local index into the frame's array
            imp = pos ? (p.gt_imp ? p.gt_imp[p.gt_off[b] + arg] : 1.f) : 1.f;
            fg = (forced || pos) && cls > 0;                        // fg_inds: labels > 0 before the bg overwrite
            if (fg) {
                gid = arg;
                encode<T>(p, static_cast<const T *>(p.gt) + (size_t)g * p.ndim, p.anchors + (size_t)a * p.ndim, tgt);
            }
        }
    }
    if (!fg)
        for (int k = 0; k < p.code; ++k) tgt[k] = 0.f;
    p.labels[o] = label;
    p.importance[o] = imp;
    if (p.gt_id) p.gt_id[o] = gid;
    if (p.overlap) p.overlap[o] = fg ? best : 0.f;
}

struct Ws {
    int *perm, *seg_off;
    void *gt_nb;
    uint32_t *gt_key;
    size_t bytes;
};

Ws carve(void *base, int batch, int num_gt, int num_segments)
{
    Ws w;
    char *p = (char *)base;
    size_t off = 0;
    const size_t g = (size_t)(num_gt > 0 ? num_gt : 1);
    w.perm = (int *)(p + off);
    off += b2s_align(sizeof(int) * g);
    w.seg_off = (int *)(p + off);
    off += b2s_align(sizeof(int) * (size_t)batch * (num_segments + 1));
    w.gt_nb = p + off;
    off += b2s_align(sizeof(double) * 4 * g);
    w.gt_key = (uint32_t *)(p + off);
    off += b2s_align(sizeof(uint32_t) * g);
    w.bytes = off;
    return w;
}

template <typename T>
int launch(const Params &p, int batch, int num_blocks, cudaStream_t stream)
{
    k_ta_gt_prep<T><<<batch, kThreads, 0, stream>>>(p);
    B2S_LAUNCH_OK();
    const dim3 grid(num_blocks, batch);
    if (p.G > 0) {
        k_ta_pass<T, false><<<grid, kThreads, 0, stream>>>(p);
        B2S_LAUNCH_OK();
    }
    k_ta_pass<T, true><<<grid, kThreads, 0, stream>>>(p);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

extern "C" size_t b2s_assign_targets_workspace_bytes(int batch, int num_gt, int num_segments)
{
    if (batch <= 0 || num_gt < 0 || num_segments <= 0) return 0;
    return carve(nullptr, batch, num_gt, num_segments).bytes;
}

extern "C" int b2s_assign_targets(const float *anchors, const float *anchor_sim, const float *matched_thr,
                                  const float *unmatched_thr, int num_anchors, int box_ndim, const int *seg_info,
                                  const double *seg_param, int num_segments, const int *blocks, int num_blocks,
                                  const void *gt_boxes, int gt_double, int num_gt, const int *gt_offsets, int batch,
                                  const int *gt_seg, const int *gt_class, const float *gt_importance,
                                  const uint8_t *anchors_mask, int code_size, int coder_flags, int *labels,
                                  float *bbox_targets, float *importance, int *gt_id, float *overlap, void *workspace,
                                  size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && batch <= 65535, "b2s_assign_targets: batch must be in [1, 65535]");
    B2S_REQUIRE(num_anchors >= 1 && num_gt >= 0, "b2s_assign_targets: num_anchors must be >= 1 and num_gt >= 0");
    B2S_REQUIRE((long long)batch * num_anchors * (code_size > 0 ? code_size : 1) < (1ll << 40),
                "b2s_assign_targets: output too large");
    B2S_REQUIRE(num_segments >= 1 && num_segments <= kMaxSegments, "b2s_assign_targets: num_segments must be 1..%d",
                kMaxSegments);
    B2S_REQUIRE(num_blocks >= 1, "b2s_assign_targets: num_blocks must be >= 1");
    B2S_REQUIRE(box_ndim >= 7, "b2s_assign_targets: box_ndim must be >= 7");
    B2S_REQUIRE((coder_flags & ~3) == 0, "b2s_assign_targets: coder_flags takes bit 0 (linear_dim), bit 1 (vec_encode)");
    B2S_REQUIRE(code_size == box_ndim + ((coder_flags & 2) ? 1 : 0),
                "b2s_assign_targets: code_size must be box_ndim (+1 with vec_encode)");
    B2S_REQUIRE(gt_double == 0 || gt_double == 1, "b2s_assign_targets: gt_double must be 0 or 1");
    B2S_REQUIRE(anchors && anchor_sim && matched_thr && unmatched_thr && seg_info && seg_param && blocks && gt_offsets,
                "b2s_assign_targets: anchor tables and gt_offsets required");
    B2S_REQUIRE(num_gt == 0 || (gt_boxes && gt_seg && gt_class), "b2s_assign_targets: gt_boxes, gt_seg, gt_class required");
    B2S_REQUIRE(labels && bbox_targets && importance && status_dev, "b2s_assign_targets: outputs and status_dev required");
    B2S_REQUIRE(((uintptr_t)anchor_sim & 15) == 0 && ((uintptr_t)seg_info & 15) == 0 && ((uintptr_t)blocks & 15) == 0,
                "b2s_assign_targets: anchor_sim, seg_info and blocks must be 16-byte aligned");
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= b2s_assign_targets_workspace_bytes(batch, num_gt, num_segments),
                "b2s_assign_targets: workspace too small");
    const Ws w = carve(workspace, batch, num_gt, num_segments);
    Params p;
    p.anchors = anchors;
    p.anchor_sim = reinterpret_cast<const float4 *>(anchor_sim);
    p.matched = matched_thr;
    p.unmatched = unmatched_thr;
    p.A = num_anchors;
    p.ndim = box_ndim;
    p.seg_info = reinterpret_cast<const int4 *>(seg_info);
    p.seg_param = seg_param;
    p.S = num_segments;
    p.blocks = reinterpret_cast<const int4 *>(blocks);
    p.gt = gt_boxes;
    p.gt_off = gt_offsets;
    p.gt_seg = gt_seg;
    p.gt_class = gt_class;
    p.gt_imp = gt_importance;
    p.G = num_gt;
    p.mask = anchors_mask;
    p.code = code_size;
    p.linear_dim = coder_flags & 1;
    p.vec_encode = (coder_flags >> 1) & 1;
    p.perm = w.perm;
    p.seg_off = w.seg_off;
    p.gt_nb = w.gt_nb;
    p.gt_key = w.gt_key;
    p.labels = labels;
    p.targets = bbox_targets;
    p.importance = importance;
    p.gt_id = gt_id;
    p.overlap = overlap;
    p.status = status_dev;
    return gt_double ? launch<double>(p, batch, num_blocks, stream) : launch<float>(p, batch, num_blocks, stream);
}
