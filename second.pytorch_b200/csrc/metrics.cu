// metrics.cu -- one training step's metrics: VoxelNet.update_metrics (second/pytorch/models/voxelnet.py:654-679) through
// torchplus/metrics.py (Accuracy, PrecisionRecall, Scalar) with the settings of every config (sigmoid scores, background
// encoded as zeros), and the per-step log figures of train.py:335-373.
//
//   k_metrics_count   one thread per (frame, anchor), grid-stride over a grid fixed by the anchor count: the anchor's
//                     sigmoid score, predicted label and threshold decisions; per-CTA integer counts (and float64 sums
//                     of the per-code localization loss) into the workspace
//   k_metrics_finish  one CTA: the partials in a fixed order into a count record (collect), then the running buffers
//                     updated in the reference's order and with its conditionals, and the record written (apply)
// b2s_train_metrics_count / _finish run the same two halves as separate launches with the count record in device
// memory between them (k_metrics_collect, k_metrics_apply), so data-parallel ranks can add their records first.
// The reference's weights are 0/1, so every tp / fp / fn / example count is an integer; they are counted as integers
// and converted to float32 once, which is exact below 2^24 per step, as torch's float32 sums of 0/1 are.  No float
// atomics; no sync.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxBlocks = 132 * 4;
constexpr int kMaxT = B2S_METRICS_MAX_THRESHOLDS;
constexpr int kMaxCode = B2S_METRICS_MAX_CODE;
constexpr int kMaxClasses = 64;

// per-CTA integer counters: unweighted correct predictions, cared anchors, cared positives, frame 0's positives,
// negatives and unmasked anchors, then tp[T] and fp[T] (cared positives / negatives scored above each threshold)
enum { I_CORRECT, I_CARED, I_POS, I_POS0, I_NEG0, I_MASK0, I_TP };
constexpr int kInts = I_TP + 2 * kMaxT;

struct Params {
    const float *cls;              // [B, A, C]
    const void *labels;            // [B, A] int32 or int64
    int labels64;
    const uint8_t *cared;          // [B, A]
    const float *loc_elem;         // [B, A, code] or null
    const uint8_t *mask;           // [B, A] or null
    int B, A, C, code, nblk;
    b2s_metrics_params p;
    const float *cls_loss, *loc_loss, *cls_pos, *cls_neg, *dir;
    b2s_metrics_buffers buf;
    float *record;
    float *counts;                 // the count record (b2s_train_metrics_count)
    int has_frame0;
    int *ipart;                    // [nblk, kInts]
    double *dpart;                 // [nblk, kMaxCode]
    unsigned *status;
};

// torch's CUDA sigmoid for float32: 1 / (1 + expf(-x)) with IEEE division and the full-precision expf
__device__ __forceinline__ float sigmoid_ref(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

__global__ void __launch_bounds__(kThreads) k_metrics_count(Params q)
{
    const int T = q.p.num_thresholds;
    const long long n = (long long)q.B * q.A;
    int cnt[I_TP] = {0, 0, 0, 0, 0, 0};
    int tp[kMaxT], fp[kMaxT];
    double le[kMaxCode];
#pragma unroll
    for (int t = 0; t < kMaxT; ++t) tp[t] = fp[t] = 0;
#pragma unroll
    for (int j = 0; j < kMaxCode; ++j) le[j] = 0.0;
    bool bad = false;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const long long label = q.labels64 ? __ldg(static_cast<const long long *>(q.labels) + i)
                                           : (long long)__ldg(static_cast<const int *>(q.labels) + i);
        bad |= label < -1 || label > q.C;
        const float *pr = q.cls + i * q.C;
        // Accuracy: argmax of the logits (first maximum; NaN wins, as torch.max) + 1 when some sigmoid passes its
        // threshold; PrecisionRecall: the largest sigmoid (NaN propagates, as torch.max)
        float best = __ldg(pr), score = sigmoid_ref(best);
        int arg = 0;
        bool any = score > q.p.acc_threshold;
        for (int c = 1; c < q.C; ++c) {
            const float v = __ldg(pr + c), s = sigmoid_ref(v);
            if (v > best || (isnan(v) && !isnan(best))) {
                best = v;
                arg = c;
            }
            if (s > score || isnan(s)) score = isnan(score) ? score : s;
            any |= s > q.p.acc_threshold;
        }
        const long long pred = any ? arg + 1 : 0;
        const bool cared = __ldg(q.cared + i) != 0;
        cnt[I_CORRECT] += pred == label;
        cnt[I_CARED] += cared;
        cnt[I_POS] += cared && label > 0;
        if (i < q.A) {
            cnt[I_POS0] += label > 0;
            cnt[I_NEG0] += label == 0;
            cnt[I_MASK0] += q.mask ? __ldg(q.mask + i) != 0 : 1;
        }
#pragma unroll
        for (int t = 0; t < kMaxT; ++t) {
            if (t < T && cared && score > q.p.thresholds[t]) {
                tp[t] += label > 0;
                fp[t] += label == 0;
            }
        }
        if (q.loc_elem) {
#pragma unroll
            for (int j = 0; j < kMaxCode; ++j)
                if (j < q.code) le[j] += (double)__ldg(q.loc_elem + i * q.code + j);
        }
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(q.status, B2S_STATUS_BAD_INPUT);

    __shared__ int s_int[kWarps][kInts];
    __shared__ double s_dbl[kWarps][kMaxCode];
#pragma unroll
    for (int c = 0; c < I_TP; ++c) {
        const int v = (int)__reduce_add_sync(0xffffffffu, (unsigned)cnt[c]);
        if (lane == 0) s_int[wid][c] = v;
    }
#pragma unroll
    for (int t = 0; t < kMaxT; ++t) {
        const int a = (int)__reduce_add_sync(0xffffffffu, (unsigned)tp[t]);
        const int b = (int)__reduce_add_sync(0xffffffffu, (unsigned)fp[t]);
        if (lane == 0) {
            s_int[wid][I_TP + t] = a;
            s_int[wid][I_TP + kMaxT + t] = b;
        }
    }
#pragma unroll
    for (int j = 0; j < kMaxCode; ++j) {
        double v = le[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_dbl[wid][j] = v;
    }
    __syncthreads();
    if (threadIdx.x < kInts) {
        int v = 0;
        for (int w = 0; w < kWarps; ++w) v += s_int[w][threadIdx.x];
        q.ipart[(size_t)blockIdx.x * kInts + threadIdx.x] = v;
    } else if (threadIdx.x >= 64 && threadIdx.x < 64 + kMaxCode) {
        const int j = threadIdx.x - 64;
        double v = 0.0;
        for (int w = 0; w < kWarps; ++w) v += s_dbl[w][j];
        q.dpart[(size_t)blockIdx.x * kMaxCode + j] = v;
    }
}

// the count record of this share (include/b2second.h, B2S_METRICS_CNT_*) from the per-CTA partials in a fixed order:
// threads 0 .. kInts-1 the integer counts, 64 .. 64+kMaxCode-1 the localization sums, kThreads-1 the frame count and
// the loss scalars.  Counts are converted to float32 once (exact below 2^24).
__device__ void collect(const Params &q, float *c)
{
    const int T = q.p.num_thresholds;
    const int i = threadIdx.x;
    if (i < kInts) {
        long long v = 0;
        for (int b = 0; b < q.nblk; ++b) v += q.ipart[(size_t)b * kInts + i];
        if (i < I_TP) {
            const bool frame0 = i == I_POS0 || i == I_NEG0 || i == I_MASK0;
            c[B2S_METRICS_CNT_CORRECT + i] = frame0 && !q.has_frame0 ? 0.f : (float)v;
        } else if (i < I_TP + T) {
            c[B2S_METRICS_COUNT_HEAD + (i - I_TP)] = (float)v;
        } else if (i >= I_TP + kMaxT && i < I_TP + kMaxT + T) {
            c[B2S_METRICS_COUNT_HEAD + T + (i - I_TP - kMaxT)] = (float)v;
        }
    } else if (i >= 64 && i < 64 + kMaxCode) {
        const int j = i - 64;
        double v = 0.0;
        for (int b = 0; b < q.nblk; ++b) v += q.dpart[(size_t)b * kMaxCode + j];
        c[B2S_METRICS_CNT_LOC_ELEM + j] = j < q.code ? (float)v : 0.f;
    } else if (i == kThreads - 1) {
        c[B2S_METRICS_CNT_FRAMES] = (float)q.B;
        c[B2S_METRICS_CNT_CLS_LOSS] = *q.cls_loss;
        c[B2S_METRICS_CNT_LOC_LOSS] = *q.loc_loss;
        c[B2S_METRICS_CNT_CLS_POS] = q.cls_pos ? *q.cls_pos : 0.f;
        c[B2S_METRICS_CNT_CLS_NEG] = q.cls_neg ? *q.cls_neg : 0.f;
        c[B2S_METRICS_CNT_DIR] = q.dir ? *q.dir : 0.f;
    }
}

// one thread: the running buffers updated from a count record in the reference's order and with its conditionals, and
// the record written.  loss_scale turns the loss slots of a record summed over W shares into the replica mean.
__device__ void apply(const float *c, const b2s_metrics_params &p, float loss_scale, const b2s_metrics_buffers &u,
                      float *r)
{
    const int T = p.num_thresholds;
    const auto loss = [&](int slot) { return loss_scale == 1.f ? c[slot] : __fmul_rn(c[slot], loss_scale); };
    // Accuracy.forward: count += clamp(sum(weights), 1), total += sum(pred == label)
    *u.acc_count = __fadd_rn(*u.acc_count, fmaxf(c[B2S_METRICS_CNT_CARED], 1.f));
    *u.acc_total = __fadd_rn(*u.acc_total, c[B2S_METRICS_CNT_CORRECT]);
    r[B2S_METRICS_REC_ACC] = __fdiv_rn(*u.acc_total, *u.acc_count);
    // PrecisionRecall.forward: per threshold, recall then precision, each only when its count is positive
    for (int t = 0; t < T; ++t) {
        const float tp = c[B2S_METRICS_COUNT_HEAD + t];
        const float fn = __fsub_rn(c[B2S_METRICS_CNT_POS], tp);
        const float fp = c[B2S_METRICS_COUNT_HEAD + T + t];
        const float rec_count = __fadd_rn(tp, fn), prec_count = __fadd_rn(tp, fp);
        if (rec_count > 0.f) {
            u.rec_count[t] = __fadd_rn(u.rec_count[t], rec_count);
            u.rec_total[t] = __fadd_rn(u.rec_total[t], tp);
        }
        if (prec_count > 0.f) {
            u.prec_count[t] = __fadd_rn(u.prec_count[t], prec_count);
            u.prec_total[t] = __fadd_rn(u.prec_total[t], tp);
        }
        // PrecisionRecall.value: totals over clamp(count, 1)
        r[B2S_METRICS_RECORD_HEAD + t] = __fdiv_rn(u.prec_total[t], fmaxf(u.prec_count[t], 1.f));
        r[B2S_METRICS_RECORD_HEAD + T + t] = __fdiv_rn(u.rec_total[t], fmaxf(u.rec_count[t], 1.f));
    }
    // Scalar.forward for the two losses: counted and added only when not 0.0 (a NaN loss is added)
    const float cl = loss(B2S_METRICS_CNT_CLS_LOSS), ll = loss(B2S_METRICS_CNT_LOC_LOSS);
    if (!(cl == 0.f)) {
        *u.cls_count = __fadd_rn(*u.cls_count, 1.f);
        *u.cls_total = __fadd_rn(*u.cls_total, cl);
    }
    if (!(ll == 0.f)) {
        *u.loc_count = __fadd_rn(*u.loc_count, 1.f);
        *u.loc_total = __fadd_rn(*u.loc_total, ll);
    }
    r[B2S_METRICS_REC_CLS] = __fdiv_rn(*u.cls_total, *u.cls_count);
    r[B2S_METRICS_REC_CLS_RT] = cl;
    r[B2S_METRICS_REC_LOC] = __fdiv_rn(*u.loc_total, *u.loc_count);
    r[B2S_METRICS_REC_LOC_RT] = ll;
    // train.py's log figures
    r[B2S_METRICS_REC_CLS_POS_RT] = loss(B2S_METRICS_CNT_CLS_POS);
    r[B2S_METRICS_REC_CLS_NEG_RT] = loss(B2S_METRICS_CNT_CLS_NEG);
    r[B2S_METRICS_REC_DIR_RT] = loss(B2S_METRICS_CNT_DIR);
    r[B2S_METRICS_REC_NUM_POS] = c[B2S_METRICS_CNT_NUM_POS];
    r[B2S_METRICS_REC_NUM_NEG] = c[B2S_METRICS_CNT_NUM_NEG];
    r[B2S_METRICS_REC_NUM_ANCHORS] = c[B2S_METRICS_CNT_NUM_ANCHORS];
    for (int j = 0; j < kMaxCode; ++j)      // loc_loss[:, :, j].sum() / batch_size
        r[B2S_METRICS_REC_LOC_ELEM + j] = __fdiv_rn(c[B2S_METRICS_CNT_LOC_ELEM + j], c[B2S_METRICS_CNT_FRAMES]);
}

constexpr int kCountFloats = B2S_METRICS_COUNT_HEAD + 2 * kMaxT;

__global__ void __launch_bounds__(kThreads) k_metrics_finish(Params q)
{
    __shared__ float s_cnt[kCountFloats];
    collect(q, s_cnt);
    __syncthreads();
    if (threadIdx.x == 0) apply(s_cnt, q.p, 1.f, q.buf, q.record);
}

__global__ void __launch_bounds__(kThreads) k_metrics_collect(Params q) { collect(q, q.counts); }

// one thread: apply's read-modify-writes of the running buffers must not be repeated by other threads
__global__ void __launch_bounds__(1) k_metrics_apply(const float *counts, b2s_metrics_params p, float loss_scale,
                                                     b2s_metrics_buffers u, float *record)
{
    if (threadIdx.x == 0) apply(counts, p, loss_scale, u, record);
}

inline int metrics_blocks(int batch, int num_anchors)
{
    const long long n = (long long)batch * num_anchors;
    const long long b = (n + kThreads - 1) / kThreads;
    return (int)(b < 1 ? 1 : (b < kMaxBlocks ? b : kMaxBlocks));
}

}  // namespace

extern "C" size_t b2s_train_metrics_workspace_bytes(int batch, int num_anchors)
{
    if (batch < 1 || num_anchors < 1) return 0;
    const size_t nblk = (size_t)metrics_blocks(batch, num_anchors);
    return b2s_align(nblk * kInts * sizeof(int)) + nblk * kMaxCode * sizeof(double);
}

namespace {

// the checks and Params of b2s_train_metrics and b2s_train_metrics_count
int count_params(const char *what, Params &q, const float *cls_preds, int num_class, const void *labels,
                 int labels_int64, const uint8_t *cared, int batch, int num_anchors, const b2s_metrics_params *params,
                 const float *cls_loss, const float *loc_loss, const float *loc_loss_elem, int code_size,
                 const uint8_t *anchors_mask, const float *cls_pos_loss, const float *cls_neg_loss,
                 const float *dir_loss, void *workspace, size_t workspace_bytes, unsigned *status_dev)
{
    B2S_REQUIRE(batch >= 1 && num_anchors >= 1 && (long long)batch * num_anchors * kMaxClasses < (1ll << 40),
                "%s: bad batch / num_anchors", what);
    B2S_REQUIRE(num_class >= 1 && num_class <= kMaxClasses, "%s: num_class must be 1..%d", what, kMaxClasses);
    B2S_REQUIRE(labels_int64 == 0 || labels_int64 == 1, "%s: labels_int64 must be 0 or 1", what);
    B2S_REQUIRE(params != nullptr && params->num_thresholds >= 1 && params->num_thresholds <= kMaxT,
                "%s: params (host) with 1..%d thresholds required", what, kMaxT);
    B2S_REQUIRE(cls_preds && labels && cared && cls_loss && loc_loss && status_dev,
                "%s: cls_preds, labels, cared, the two losses and status_dev required", what);
    B2S_REQUIRE(loc_loss_elem == nullptr || (code_size >= 1 && code_size <= kMaxCode),
                "%s: code_size must be 1..%d with loc_loss_elem", what, kMaxCode);
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= b2s_train_metrics_workspace_bytes(batch, num_anchors),
                "%s: workspace too small", what);
    q = Params{};
    q.cls = cls_preds;
    q.labels = labels;
    q.labels64 = labels_int64;
    q.cared = cared;
    q.loc_elem = loc_loss_elem;
    q.mask = anchors_mask;
    q.B = batch;
    q.A = num_anchors;
    q.C = num_class;
    q.code = loc_loss_elem ? code_size : 0;
    q.nblk = metrics_blocks(batch, num_anchors);
    q.p = *params;
    q.cls_loss = cls_loss;
    q.loc_loss = loc_loss;
    q.cls_pos = cls_pos_loss;
    q.cls_neg = cls_neg_loss;
    q.dir = dir_loss;
    q.has_frame0 = 1;
    q.ipart = static_cast<int *>(workspace);
    q.dpart = reinterpret_cast<double *>(static_cast<char *>(workspace) + b2s_align((size_t)q.nblk * kInts * sizeof(int)));
    q.status = status_dev;
    return 0;
}

int check_buffers(const char *what, const b2s_metrics_buffers *buffers)
{
    B2S_REQUIRE(buffers != nullptr && buffers->acc_total && buffers->acc_count && buffers->prec_total &&
                    buffers->prec_count && buffers->rec_total && buffers->rec_count && buffers->cls_total &&
                    buffers->cls_count && buffers->loc_total && buffers->loc_count,
                "%s: all ten running buffers required", what);
    return 0;
}

}  // namespace

extern "C" int b2s_train_metrics(const float *cls_preds, int num_class, const void *labels, int labels_int64,
                                 const uint8_t *cared, int batch, int num_anchors, const b2s_metrics_params *params,
                                 const float *cls_loss, const float *loc_loss, const float *loc_loss_elem, int code_size,
                                 const uint8_t *anchors_mask, const float *cls_pos_loss, const float *cls_neg_loss,
                                 const float *dir_loss, const b2s_metrics_buffers *buffers, float *record,
                                 void *workspace, size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    const char *what = "b2s_train_metrics";
    Params q;
    if (int e = count_params(what, q, cls_preds, num_class, labels, labels_int64, cared, batch, num_anchors, params,
                             cls_loss, loc_loss, loc_loss_elem, code_size, anchors_mask, cls_pos_loss, cls_neg_loss,
                             dir_loss, workspace, workspace_bytes, status_dev))
        return e;
    B2S_REQUIRE(record != nullptr, "%s: record required", what);
    if (int e = check_buffers(what, buffers)) return e;
    cudaStream_t stream = (cudaStream_t)stream_;
    q.buf = *buffers;
    q.record = record;
    k_metrics_count<<<q.nblk, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    k_metrics_finish<<<1, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_train_metrics_count(const float *cls_preds, int num_class, const void *labels, int labels_int64,
                                       const uint8_t *cared, int batch, int num_anchors,
                                       const b2s_metrics_params *params, const float *cls_loss, const float *loc_loss,
                                       const float *loc_loss_elem, int code_size, const uint8_t *anchors_mask,
                                       const float *cls_pos_loss, const float *cls_neg_loss, const float *dir_loss,
                                       int has_frame0, float *counts, void *workspace, size_t workspace_bytes,
                                       unsigned *status_dev, void *stream_)
{
    const char *what = "b2s_train_metrics_count";
    Params q;
    if (int e = count_params(what, q, cls_preds, num_class, labels, labels_int64, cared, batch, num_anchors, params,
                             cls_loss, loc_loss, loc_loss_elem, code_size, anchors_mask, cls_pos_loss, cls_neg_loss,
                             dir_loss, workspace, workspace_bytes, status_dev))
        return e;
    B2S_REQUIRE(counts != nullptr && (has_frame0 == 0 || has_frame0 == 1),
                "%s: counts required, has_frame0 must be 0 or 1", what);
    cudaStream_t stream = (cudaStream_t)stream_;
    q.has_frame0 = has_frame0;
    q.counts = counts;
    k_metrics_count<<<q.nblk, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    k_metrics_collect<<<1, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_train_metrics_finish(const float *counts, const b2s_metrics_params *params, float loss_scale,
                                        const b2s_metrics_buffers *buffers, float *record, void *stream_)
{
    const char *what = "b2s_train_metrics_finish";
    B2S_REQUIRE(params != nullptr && params->num_thresholds >= 1 && params->num_thresholds <= kMaxT,
                "%s: params (host) with 1..%d thresholds required", what, kMaxT);
    B2S_REQUIRE(counts != nullptr && record != nullptr, "%s: counts and record required", what);
    B2S_REQUIRE(isfinite(loss_scale) && loss_scale > 0.f, "%s: loss_scale must be finite and positive", what);
    if (int e = check_buffers(what, buffers)) return e;
    k_metrics_apply<<<1, 1, 0, (cudaStream_t)stream_>>>(counts, *params, loss_scale, *buffers, record);
    B2S_LAUNCH_OK();
    return 0;
}
