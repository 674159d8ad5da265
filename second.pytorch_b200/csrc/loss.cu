// loss.cu -- VoxelNet.loss (second/pytorch/models/voxelnet.py:239-312) with the settings of every config: sigmoid focal
// classification (losses.py:236-294), smooth-L1 localization with the sin encoding of the yaw (voxelnet.py:704-753,
// losses.py:135-182), NormByNumPositives weights (voxelnet.py:756-795) and the softmax direction classifier
// (voxelnet.py:284-297,814-828), and its gradient.
//
//   k_loss_count   one thread per (frame, anchor): per-CTA positive count and sum of positive importance (the two
//                  per-frame normalizers), bad labels
//   k_loss_fwd     one thread per (frame, anchor): each CTA first reduces its frame's count partials in a fixed order
//                  (every CTA of the frame gets the same bits), then the anchor's focal, smooth-L1 and softmax terms;
//                  per-anchor outputs and per-CTA partial sums in float64
//   k_loss_finish  one CTA: the partial sums in a fixed order -> the six scalars
//   k_loss_bwd     one thread per (frame, anchor): d box, d cls, d dir from the frame's normalizers and the incoming
//                  gradients of the four differentiable scalars
// No float atomics anywhere: every sum has one order, so results are bit-reproducible.  Per-anchor terms are float32;
// the sums over anchors accumulate in float64 and are rounded once.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kCode = 7;
constexpr int kMaxClasses = 64;
constexpr int kMaxBins = 16;
constexpr int kParts = 5;           // per-CTA partial sums: cls, loc, dir, cls_pos, cls_neg

struct Params {
    const float *box, *cls, *dir;  // [B, A, 7], [B, A, C], [B, A, nb]
    const void *labels;            // [B, A] int32 or int64
    int labels64;
    const float *reg, *imp, *anchors;   // [B, A, 7], [B, A], [B, A, 7]
    int B, A, C, nb, nblk;
    b2s_loss_params p;
    float thr;                     // 1 / sigma^2 and 0.5 / sigma^2 as the reference's float32 scalars compare them
    float half_thr;
    float period, bin_width;       // 2 pi and 2 pi / nb in float32
    int2 *count_part;              // [B, nblk]: (positives, 0)
    double *imp_part;              // [B, nblk]: sum of positive importance
    double *loss_part;             // [B * nblk, kParts]
    float *norms;                  // [B, 2]: max(positives, 1), max(sum of positive importance, 1)
    float *reduced, *pos_neg;      // [4], [2]
    float *cls_loss, *loc_loss;    // optional [B, A, C], [B, A, 7]
    uint8_t *cared;                // optional [B, A]
    const float *dred;             // [4] or null
    float *dbox, *dcls, *ddir;
    unsigned *status;
};

// the anchor's label; a label outside [-1, C] reads as -1 (not cared)
__device__ __forceinline__ int load_label(const Params &q, size_t o, bool *bad)
{
    const long long l = q.labels64 ? static_cast<const long long *>(q.labels)[o]
                                   : (long long)static_cast<const int *>(q.labels)[o];
    *bad = l < -1 || l > q.C;
    return *bad ? -1 : (int)l;
}

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

__device__ __forceinline__ int warp_sum(int v)
{
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// limit_period(rot - dir_offset, 0, 2 pi) binned into nb bins (get_direction_target), each step one float32 rounding
// as torch runs it on float32 tensors with Python-float scalars
__device__ __forceinline__ int direction_bin(const Params &q, float t6, float a6)
{
    const float x = __fsub_rn(__fadd_rn(t6, a6), q.p.dir_offset);
    const float lp = __fsub_rn(x, __fmul_rn(floorf(__fdiv_rn(x, q.period)), q.period));
    const int bin = (int)floorf(__fdiv_rn(lp, q.bin_width));
    return min(max(bin, 0), q.nb - 1);
}

// the frame's two normalizers from its count partials, summed in a fixed order by warp 0; every CTA gets the same bits
__device__ __forceinline__ float2 frame_norms(const Params &q, int b, float2 *s_norm)
{
    if (threadIdx.x < 32) {
        int n = 0;
        double w = 0.0;
        for (int i = threadIdx.x; i < q.nblk; i += 32) {
            n += q.count_part[(size_t)b * q.nblk + i].x;
            w += q.imp_part[(size_t)b * q.nblk + i];
        }
        n = warp_sum(n);
        w = warp_sum(w);
        if (threadIdx.x == 0) *s_norm = make_float2(fmaxf((float)n, 1.f), fmaxf(__double2float_rn(w), 1.f));
    }
    __syncthreads();
    return *s_norm;
}

__global__ void __launch_bounds__(kThreads) k_loss_count(Params q)
{
    __shared__ int s_n[kWarps];
    __shared__ double s_w[kWarps];
    const int b = blockIdx.y, a = blockIdx.x * kThreads + threadIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int pos = 0;
    double w = 0.0;
    bool bad = false;
    if (a < q.A) {
        const size_t o = (size_t)b * q.A + a;
        const int l = load_label(q, o, &bad);
        pos = l > 0;
        w = pos ? (double)q.imp[o] : 0.0;
    }
    if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(q.status, B2S_STATUS_BAD_INPUT);
    pos = warp_sum(pos);
    w = warp_sum(w);
    if (lane == 0) {
        s_n[wid] = pos;
        s_w[wid] = w;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = 0;
        double t = 0.0;
        for (int i = 0; i < kWarps; ++i) {
            n += s_n[i];
            t += s_w[i];
        }
        q.count_part[(size_t)b * q.nblk + blockIdx.x] = make_int2(n, 0);
        q.imp_part[(size_t)b * q.nblk + blockIdx.x] = t;
    }
}

// softplus(-|x|) = log1p(exp(-|x|)) and the two sigmoids from e = exp(-|x|), none of which overflows
struct Sig {
    float ce_tail, p, q;           // log1p(e), sigmoid(x), 1 - sigmoid(x)
};

__device__ __forceinline__ Sig sigmoid_parts(float x)
{
    const float e = expf(-fabsf(x));
    const float r = 1.f / (1.f + e);
    Sig s;
    s.ce_tail = log1pf(e);
    s.p = x >= 0.f ? r : e * r;
    s.q = x >= 0.f ? e * r : r;
    return s;
}

// focal term (p_t and the alpha factor spelled out for z in {0, 1}) without the anchor weight
__device__ __forceinline__ float focal(const Params &q, float x, bool z, const Sig &s)
{
    const float ce = fmaxf(x, 0.f) - (z ? x : 0.f) + s.ce_tail;
    const float omp = z ? s.q : s.p;                                 // 1 - p_t
    const float m = q.p.gamma == 2.f ? omp * omp : powf(omp, q.p.gamma);
    return m * (z ? q.p.alpha : 1.f - q.p.alpha) * ce;
}

// d focal / dx without the anchor weight: z = 1: alpha (1-p)^g (dCE - g p CE); z = 0: (1-alpha) p^g (g (1-p) CE + dCE)
// with dCE = p - z.  At x == 0 exactly the reference's autograd takes clamp's subgradient 1 and abs's 0, so dCE = 1 - z
// there; that is kept.
__device__ __forceinline__ float focal_grad(const Params &q, float x, bool z, const Sig &s)
{
    const float ce = fmaxf(x, 0.f) - (z ? x : 0.f) + s.ce_tail;
    const float omp = z ? s.q : s.p;                                 // 1 - p_t
    const float m = q.p.gamma == 2.f ? omp * omp : powf(omp, q.p.gamma);
    const float dce = x == 0.f ? (z ? 0.f : 1.f) : (z ? -s.q : s.p);
    return z ? q.p.alpha * m * (dce - q.p.gamma * s.p * ce) : (1.f - q.p.alpha) * m * (q.p.gamma * s.q * ce + dce);
}

// smooth-L1 of d = cw * (pred - target) (the yaw component sin-encoded) and its derivative in d
__device__ __forceinline__ float smooth_l1(const Params &q, float d, float *dd)
{
    const float ad = fabsf(d);
    const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
    if (ad <= q.thr) {
        const float s = ad * q.p.sigma;
        *dd = sg * q.p.sigma * s;
        return 0.5f * s * s;
    }
    *dd = sg;
    return ad - q.half_thr;
}

// the box difference of component k with its d(pred) factor: the yaw is sin(f p) cos(f t) - cos(f p) sin(f t)
// = sin(f (p - t)), whose derivative in p is f cos(f (p - t)).  f (p - t) is formed in float64 (the float products
// are exact there): rounded to float32 it would carry an absolute error of eps32 |p - t|, which the sine keeps as is
// when p - t is near a multiple of pi
__device__ __forceinline__ float box_diff(const Params &q, const float *bp, const float *rt, int k, float *dk)
{
    const float cw = q.p.code_weight[k];
    if (k == 6) {
        const double f = q.p.sin_factor;
        const double u = __dsub_rn(__dmul_rn(f, (double)bp[6]), __dmul_rn(f, (double)rt[6]));
        double su, cu;
        sincos(u, &su, &cu);
        *dk = cw * __double2float_rn(f * cu);
        return cw * __double2float_rn(su);
    }
    *dk = cw;
    return cw * (bp[k] - rt[k]);
}

struct AnchorW {
    int label, bin;
    float cls_w, reg_w, dir_w;
};

__device__ __forceinline__ AnchorW anchor_weights(const Params &q, size_t o, float2 nrm)
{
    AnchorW w;
    bool bad;
    w.label = load_label(q, o, &bad);
    const bool pos = w.label > 0, neg = w.label == 0;
    const float imp = q.imp[o];
    // ((neg * w_neg + w_pos * pos) / max(npos, 1)) * importance, (pos / max(npos, 1)) * importance
    const float cw = (neg ? q.p.neg_cls_weight : 0.f) + (pos ? q.p.pos_cls_weight : 0.f);
    w.cls_w = __fdiv_rn(cw, nrm.x) * imp;
    w.reg_w = __fdiv_rn(pos ? 1.f : 0.f, nrm.x) * imp;
    w.dir_w = pos ? __fdiv_rn(imp, nrm.y) : 0.f;
    w.bin = pos ? direction_bin(q, q.reg[o * kCode + 6], q.anchors[o * kCode + 6]) : 0;
    return w;
}

// softmax cross-entropy of the anchor's direction logits against bin `bin`, and log-sum-exp pieces for the gradient
__device__ __forceinline__ float dir_ce(const Params &q, const float *dl, int bin, float *mx, float *se)
{
    float m = dl[0];
    for (int j = 1; j < q.nb; ++j) m = fmaxf(m, dl[j]);
    float s = 0.f;
    for (int j = 0; j < q.nb; ++j) s += expf(dl[j] - m);
    *mx = m;
    *se = s;
    return logf(s) + m - dl[bin];
}

__global__ void __launch_bounds__(kThreads) k_loss_fwd(Params q)
{
    __shared__ float2 s_norm;
    __shared__ double s_part[kWarps][kParts];
    const int b = blockIdx.y, a = blockIdx.x * kThreads + threadIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const float2 nrm = frame_norms(q, b, &s_norm);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        q.norms[2 * b] = nrm.x;
        q.norms[2 * b + 1] = nrm.y;
    }
    double part[kParts] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (a < q.A) {
        const size_t o = (size_t)b * q.A + a;
        const AnchorW w = anchor_weights(q, o, nrm);
        // classification: every class column; the cls_pos / cls_neg split of _get_pos_neg_loss (voxelnet.py:20-34)
        const float *x = q.cls + o * q.C;
        double col0 = 0.0, rest = 0.0;
        for (int c = 0; c < q.C; ++c) {
            const float v = x[c];
            const bool z = w.label == c + 1;
            const float l = focal(q, v, z, sigmoid_parts(v)) * w.cls_w;
            if (q.cls_loss) q.cls_loss[o * q.C + c] = l;
            if (c == 0) col0 = l;
            else rest += l;
        }
        part[0] = col0 + rest;
        if (q.C == 1) {
            part[3] = w.label > 0 ? col0 : 0.0;
            part[4] = w.label == 0 ? col0 : 0.0;
        } else {                                                     // the reference's columns 1: and column 0
            part[3] = rest;
            part[4] = col0;
        }
        // localization
        const float *bp = q.box + o * kCode, *rt = q.reg + o * kCode;
        double loc_sum = 0.0;
#pragma unroll
        for (int k = 0; k < kCode; ++k) {
            float dk, dd;
            const float l = smooth_l1(q, box_diff(q, bp, rt, k, &dk), &dd) * w.reg_w;
            if (q.loc_loss) q.loc_loss[o * kCode + k] = l;
            loc_sum += l;
        }
        part[1] = loc_sum;
        // direction
        if (w.dir_w != 0.f) {
            float mx, se;
            part[2] = dir_ce(q, q.dir + o * q.nb, w.bin, &mx, &se) * w.dir_w;
        }
        if (q.cared) q.cared[o] = w.label >= 0;
    }
#pragma unroll
    for (int k = 0; k < kParts; ++k) {
        const double v = warp_sum(part[k]);
        if (lane == 0) s_part[wid][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < kParts) {
        double t = 0.0;
        for (int i = 0; i < kWarps; ++i) t += s_part[i][threadIdx.x];
        q.loss_part[((size_t)b * q.nblk + blockIdx.x) * kParts + threadIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kThreads) k_loss_finish(Params q)
{
    __shared__ double s_part[kWarps][kParts];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t n = (size_t)q.B * q.nblk;
    double t[kParts] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (size_t i = threadIdx.x; i < n; i += kThreads)
#pragma unroll
        for (int k = 0; k < kParts; ++k) t[k] += q.loss_part[i * kParts + k];
#pragma unroll
    for (int k = 0; k < kParts; ++k) {
        const double v = warp_sum(t[k]);
        if (lane == 0) s_part[wid][k] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s[kParts];
        for (int k = 0; k < kParts; ++k) {
            s[k] = 0.0;
            for (int i = 0; i < kWarps; ++i) s[k] += s_part[i][k];
        }
        const float B = (float)q.B;
        // the reference's order: sum / batch, then * weight; loss = loc + cls, then += dir * w_dir
        const float cls_red = (__double2float_rn(s[0]) / B) * q.p.cls_weight;
        const float loc_red = (__double2float_rn(s[1]) / B) * q.p.loc_weight;
        const float dir_red = __double2float_rn(s[2]) / B;
        q.reduced[0] = loc_red + cls_red + dir_red * q.p.dir_weight;
        q.reduced[1] = cls_red;
        q.reduced[2] = loc_red;
        q.reduced[3] = dir_red;
        q.pos_neg[0] = (__double2float_rn(s[3]) / B) / q.p.pos_cls_weight;
        q.pos_neg[1] = (__double2float_rn(s[4]) / B) / q.p.neg_cls_weight;
    }
}

__global__ void __launch_bounds__(kThreads) k_loss_bwd(Params q)
{
    const int b = blockIdx.y, a = blockIdx.x * kThreads + threadIdx.x;
    if (a >= q.A) return;
    const size_t o = (size_t)b * q.A + a;
    const float2 nrm = make_float2(q.norms[2 * b], q.norms[2 * b + 1]);
    const float g_loss = q.dred ? q.dred[0] : 0.f, g_cls = q.dred ? q.dred[1] : 0.f;
    const float g_loc = q.dred ? q.dred[2] : 0.f, g_dir = q.dred ? q.dred[3] : 0.f;
    const float B = (float)q.B;
    const AnchorW w = anchor_weights(q, o, nrm);
    // classification
    const float gc = (g_loss + g_cls) * q.p.cls_weight / B * w.cls_w;
    const float *x = q.cls + o * q.C;
    float *dx = q.dcls + o * q.C;
    for (int c = 0; c < q.C; ++c) {
        const float v = x[c];
        dx[c] = w.cls_w == 0.f ? 0.f : gc * focal_grad(q, v, w.label == c + 1, sigmoid_parts(v));
    }
    // localization
    const float gl = (g_loss + g_loc) * q.p.loc_weight / B * w.reg_w;
    const float *bp = q.box + o * kCode, *rt = q.reg + o * kCode;
    float *db = q.dbox + o * kCode;
#pragma unroll
    for (int k = 0; k < kCode; ++k) {
        if (w.reg_w == 0.f) {
            db[k] = 0.f;
            continue;
        }
        float dk, dd;
        smooth_l1(q, box_diff(q, bp, rt, k, &dk), &dd);
        db[k] = gl * dd * dk;
    }
    // direction: (softmax - one-hot) * weight
    const float *dl = q.dir + o * q.nb;
    float *dd = q.ddir + o * q.nb;
    if (w.dir_w == 0.f) {
        for (int j = 0; j < q.nb; ++j) dd[j] = 0.f;
        return;
    }
    const float gd = (g_loss * q.p.dir_weight + g_dir) / B * w.dir_w;
    float mx, se;
    dir_ce(q, dl, w.bin, &mx, &se);
    for (int j = 0; j < q.nb; ++j) dd[j] = gd * (expf(dl[j] - mx) / se - (j == w.bin ? 1.f : 0.f));
}

struct Ws {
    int2 *count_part;
    double *imp_part, *loss_part;
    size_t bytes;
};

Ws carve(void *base, int batch, int num_anchors)
{
    const size_t n = (size_t)batch * b2s_cdiv(num_anchors, kThreads);
    char *p = (char *)base;
    Ws w;
    size_t off = 0;
    w.count_part = (int2 *)(p + off);
    off += b2s_align(sizeof(int2) * n);
    w.imp_part = (double *)(p + off);
    off += b2s_align(sizeof(double) * n);
    w.loss_part = (double *)(p + off);
    off += b2s_align(sizeof(double) * kParts * n);
    w.bytes = off;
    return w;
}

int fill(Params &q, const float *box, const float *cls, const float *dir, int num_class, int num_bins,
         const void *labels, int labels_int64, const float *reg, const float *imp, const float *anchors, int batch,
         int num_anchors, const b2s_loss_params *params, const char *what)
{
    B2S_REQUIRE(batch >= 1 && batch <= 65535, "%s: batch must be in [1, 65535]", what);
    B2S_REQUIRE(num_anchors >= 1 && (long long)num_anchors * kMaxClasses < (1ll << 31),
                "%s: num_anchors must be in [1, 2^25)", what);
    B2S_REQUIRE(num_class >= 1 && num_class <= kMaxClasses, "%s: num_class must be 1..%d", what, kMaxClasses);
    B2S_REQUIRE(num_bins >= 1 && num_bins <= kMaxBins, "%s: num_dir_bins must be 1..%d", what, kMaxBins);
    B2S_REQUIRE(labels_int64 == 0 || labels_int64 == 1, "%s: labels_int64 must be 0 or 1", what);
    B2S_REQUIRE(params != nullptr, "%s: params (host) required", what);
    B2S_REQUIRE(params->num_dir_bins == num_bins, "%s: params->num_dir_bins disagrees with num_dir_bins", what);
    B2S_REQUIRE(params->sigma > 0.f && params->pos_cls_weight != 0.f && params->neg_cls_weight != 0.f,
                "%s: sigma must be > 0 and the class weights nonzero", what);
    B2S_REQUIRE(box && cls && dir && labels && reg && imp && anchors, "%s: inputs required", what);
    q = Params{};
    q.box = box;
    q.cls = cls;
    q.dir = dir;
    q.labels = labels;
    q.labels64 = labels_int64;
    q.reg = reg;
    q.imp = imp;
    q.anchors = anchors;
    q.B = batch;
    q.A = num_anchors;
    q.C = num_class;
    q.nb = num_bins;
    q.nblk = b2s_cdiv(num_anchors, kThreads);
    q.p = *params;
    const double s2 = (double)params->sigma * params->sigma;
    q.thr = (float)(1.0 / s2);
    q.half_thr = (float)(0.5 / s2);
    q.period = (float)(2.0 * M_PI);
    q.bin_width = (float)(2.0 * M_PI / num_bins);
    return 0;
}

}  // namespace

extern "C" size_t b2s_detection_loss_workspace_bytes(int batch, int num_anchors)
{
    if (batch <= 0 || num_anchors <= 0) return 0;
    return carve(nullptr, batch, num_anchors).bytes;
}

extern "C" int b2s_detection_loss(const float *box_preds, const float *cls_preds, const float *dir_preds,
                                  int num_class, int num_dir_bins, const void *labels, int labels_int64,
                                  const float *reg_targets, const float *importance, const float *anchors, int batch,
                                  int num_anchors, const b2s_loss_params *params, float *reduced, float *pos_neg,
                                  float *cls_loss, float *loc_loss, uint8_t *cared, float *norms, void *workspace,
                                  size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    const char *what = "b2s_detection_loss";
    cudaStream_t stream = (cudaStream_t)stream_;
    Params q;
    const int rc = fill(q, box_preds, cls_preds, dir_preds, num_class, num_dir_bins, labels, labels_int64, reg_targets,
                        importance, anchors, batch, num_anchors, params, what);
    if (rc) return rc;
    B2S_REQUIRE(reduced && pos_neg && norms && status_dev, "%s: reduced, pos_neg, norms and status_dev required", what);
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= b2s_detection_loss_workspace_bytes(batch, num_anchors),
                "%s: workspace too small", what);
    const Ws w = carve(workspace, batch, num_anchors);
    q.count_part = w.count_part;
    q.imp_part = w.imp_part;
    q.loss_part = w.loss_part;
    q.norms = norms;
    q.reduced = reduced;
    q.pos_neg = pos_neg;
    q.cls_loss = cls_loss;
    q.loc_loss = loc_loss;
    q.cared = cared;
    q.status = status_dev;
    const dim3 grid(q.nblk, batch);
    k_loss_count<<<grid, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    k_loss_fwd<<<grid, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    k_loss_finish<<<1, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_detection_loss_backward(const float *box_preds, const float *cls_preds, const float *dir_preds,
                                           int num_class, int num_dir_bins, const void *labels, int labels_int64,
                                           const float *reg_targets, const float *importance, const float *anchors,
                                           int batch, int num_anchors, const b2s_loss_params *params,
                                           const float *norms, const float *d_reduced, float *d_box, float *d_cls,
                                           float *d_dir, void *stream_)
{
    const char *what = "b2s_detection_loss_backward";
    cudaStream_t stream = (cudaStream_t)stream_;
    Params q;
    const int rc = fill(q, box_preds, cls_preds, dir_preds, num_class, num_dir_bins, labels, labels_int64, reg_targets,
                        importance, anchors, batch, num_anchors, params, what);
    if (rc) return rc;
    B2S_REQUIRE(norms && d_box && d_cls && d_dir, "%s: norms and the three gradients required", what);
    q.norms = const_cast<float *>(norms);
    q.dred = d_reduced;
    q.dbox = d_box;
    q.dcls = d_cls;
    q.ddir = d_dir;
    k_loss_bwd<<<dim3(q.nblk, batch), kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    return 0;
}
