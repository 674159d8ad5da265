// optim.cu -- the optimizer step of second/pytorch/train.py:299,323-325 for every parameter tensor at once:
// torch.nn.utils.clip_grad_norm_(net.parameters(), 10.0), OptimWrapper.step (torchplus/train/fastai_optim.py:154-167:
// the decoupled decay p *= 1 - wd * lr of fixed_weight_decay, then torch.optim.Adam.step, or Adam with its L2 decay
// g += wd * p), the learning-rate / momentum schedule of LRSchedulerStep.step
// (torchplus/train/learning_schedules_fastai.py:43-56) and zero_grad.
//
//   k_opt_norm   one CTA per chunk of kChunk elements of one tensor (the chunk table is built once by the caller):
//                the chunk's sum of g^2 as one float64 partial; CTA 0 also latches the step counter for the next kernel
//   k_opt_step   the same chunks: each CTA first adds all partials in one fixed order (every CTA gets the same bits of
//                the norm and the clip coefficient), reads the step's row of the hyper-parameter table, then clips,
//                decays and updates m, v, p of its chunk and zeroes g; CTA 0 stores the norm and advances the counter
// No float atomics: every sum has one order, so two calls on the same inputs give the same bits.  Every float32 step
// of the update is an explicit round-to-nearest intrinsic in the order written in adam_element (no FMA contraction),
// and the vector and scalar paths share it, so a value's result does not depend on where its tensor starts or ends.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = B2S_OPTIM_CHUNK;
constexpr int kCols = B2S_OPTIM_HYPER_COLS;

struct Params {
    float *const *p;
    float *const *g;
    float *const *m;
    float *const *v;
    int num_tensors;
    const int4 *chunks;            // [num_chunks]: (tensor, first element, elements, 0)
    int num_chunks;
    const double *hyper;           // [total_step, kCols]: lr, beta1, 1 - beta1^t, sqrt(1 - beta2^t), 1 - wd * lr
    long long total_step;
    long long *step;               // steps taken so far; row min(step, total_step - 1) is the one applied
    long long *step_now;           // workspace: the counter as k_opt_norm found it
    double *part;                  // workspace [num_chunks]
    int decoupled, zero_grad;
    float wd, beta2, one_minus_beta2, eps, max_norm;
    float *total_norm;
    unsigned *status;
};

// what one step needs beyond the element's own p, g, m, v; the same bits in every thread of every CTA
struct Step {
    float coef;                    // min(1, max_norm / (norm + 1e-6)), NaN when the norm is
    float decay;                   // 1 - wd * lr (decoupled form)
    float one_minus_beta1;
    float step_size;               // lr / (1 - beta1^t)
    float bc2_sqrt;                // sqrt(1 - beta2^t)
    float norm;
};

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    return v;
}

// the sum of `v` over the CTA in one fixed order; valid in thread 0
__device__ __forceinline__ double block_sum(double v, double *s_warp)
{
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int i = 0; i < kWarps; ++i) t += s_warp[i];
    return t;
}

__device__ __forceinline__ bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// a chunk whose tensor index, offset or count cannot be right is skipped (and reported): nothing is read through it
__device__ __forceinline__ bool chunk_ok(const Params &q, const int4 c)
{
    return c.x >= 0 && c.x < q.num_tensors && c.y >= 0 && c.z >= 0 && c.z <= kChunk;
}

__global__ void __launch_bounds__(kThreads) k_opt_norm(Params q)
{
    __shared__ double s_warp[kWarps];
    if (blockIdx.x == 0 && threadIdx.x == 0) *q.step_now = *q.step;
    const int4 c = q.chunks[blockIdx.x];
    double acc = 0.0;                                                // g * g is exact in float64
    const float *g = chunk_ok(q, c) ? q.g[c.x] : nullptr;
    if (g != nullptr) {
        g += c.y;
        const int n4 = aligned16(g) ? c.z / 4 : 0;
        const float4 *g4 = reinterpret_cast<const float4 *>(g);
        for (int i = threadIdx.x; i < n4; i += kThreads) {
            const float4 x = g4[i];
            acc += (double)x.x * x.x;
            acc += (double)x.y * x.y;
            acc += (double)x.z * x.z;
            acc += (double)x.w * x.w;
        }
        for (int i = n4 * 4 + threadIdx.x; i < c.z; i += kThreads) acc += (double)g[i] * g[i];
    }
    const double t = block_sum(acc, s_warp);
    if (threadIdx.x == 0) q.part[blockIdx.x] = t;
}

// clip -> decay -> moments -> parameter, each line one float32 rounding (torch's op chain on float32 tensors with the
// Python-double scalars rounded to float32 first)
__device__ __forceinline__ void adam_element(const Params &q, const Step &s, float &p, float g, float &m, float &v)
{
    g = __fmul_rn(g, s.coef);                                        // g.mul_(clip_coef_clamped)
    if (q.decoupled) p = __fmul_rn(p, s.decay);                      // p.mul_(1 - wd * lr)
    else g = __fadd_rn(g, __fmul_rn(q.wd, p));                       // grad.add(p, alpha=wd)
    m = __fadd_rn(m, __fmul_rn(__fsub_rn(g, m), s.one_minus_beta1)); // exp_avg.lerp_(grad, 1 - beta1)
    v = __fadd_rn(__fmul_rn(q.beta2, v), __fmul_rn(__fmul_rn(q.one_minus_beta2, g), g));
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), s.bc2_sqrt), q.eps);
    p = __fsub_rn(p, __fmul_rn(s.step_size, __fdiv_rn(m, denom)));   // p.addcdiv_(exp_avg, denom, value=-step_size)
}

__global__ void __launch_bounds__(kThreads) k_opt_step(Params q)
{
    __shared__ double s_warp[kWarps];
    __shared__ Step s_step;
    {
        double acc = 0.0;
        for (int i = threadIdx.x; i < q.num_chunks; i += kThreads) acc += q.part[i];
        const double sum = block_sum(acc, s_warp);
        if (threadIdx.x == 0) {
            const long long now = *q.step_now;
            const long long row = now < 0 ? 0 : (now < q.total_step ? now : q.total_step - 1);
            const double *h = q.hyper + row * kCols;
            Step s;
            s.norm = __double2float_rn(sqrt(sum));
            const float coef = __fdiv_rn(q.max_norm, __fadd_rn(s.norm, 1e-6f));
            s.coef = coef > 1.f ? 1.f : coef;                        // keeps a NaN, as torch.clamp does
            s.decay = __double2float_rn(h[4]);
            s.one_minus_beta1 = __double2float_rn(__dsub_rn(1.0, h[1]));
            s.step_size = __double2float_rn(__ddiv_rn(h[0], h[2]));
            s.bc2_sqrt = __double2float_rn(h[3]);
            s_step = s;
            if (blockIdx.x == 0) {
                *q.total_norm = s.norm;
                *q.step = now + 1;
                unsigned bits = 0;
                if (!isfinite(s.norm)) bits |= B2S_STATUS_OPT_NONFINITE;
                if (now < 0 || now >= q.total_step) bits |= B2S_STATUS_BAD_INPUT;
                if (bits) atomicOr(q.status, bits);
            }
        }
        __syncthreads();
    }
    const Step s = s_step;
    const int4 c = q.chunks[blockIdx.x];
    if (!chunk_ok(q, c)) {
        if (threadIdx.x == 0) atomicOr(q.status, B2S_STATUS_BAD_INPUT);
        return;
    }
    float *p = q.p[c.x] + c.y;
    float *g = q.g[c.x];
    if (g == nullptr) {                                              // no gradient: decayed (decoupled form), not stepped
        if (q.decoupled)
            for (int i = threadIdx.x; i < c.z; i += kThreads) p[i] = __fmul_rn(p[i], s.decay);
        return;
    }
    g += c.y;
    float *m = q.m[c.x] + c.y, *v = q.v[c.x] + c.y;
    const int n4 = aligned16(p) && aligned16(g) && aligned16(m) && aligned16(v) ? c.z / 4 : 0;
    float4 *p4 = reinterpret_cast<float4 *>(p), *g4 = reinterpret_cast<float4 *>(g);
    float4 *m4 = reinterpret_cast<float4 *>(m), *v4 = reinterpret_cast<float4 *>(v);
#pragma unroll 2
    for (int i = threadIdx.x; i < n4; i += kThreads) {
        float4 pp = p4[i], mm = m4[i], vv = v4[i];
        const float4 gg = g4[i];
        adam_element(q, s, pp.x, gg.x, mm.x, vv.x);
        adam_element(q, s, pp.y, gg.y, mm.y, vv.y);
        adam_element(q, s, pp.z, gg.z, mm.z, vv.z);
        adam_element(q, s, pp.w, gg.w, mm.w, vv.w);
        p4[i] = pp;
        m4[i] = mm;
        v4[i] = vv;
        if (q.zero_grad) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int i = n4 * 4 + threadIdx.x; i < c.z; i += kThreads) {
        adam_element(q, s, p[i], g[i], m[i], v[i]);
        if (q.zero_grad) g[i] = 0.f;
    }
}

struct Ws {
    double *part;
    long long *step_now;
    size_t bytes;
};

Ws carve(void *base, int num_chunks)
{
    char *p = (char *)base;
    Ws w;
    size_t off = 0;
    w.part = (double *)(p + off);
    off += b2s_align(sizeof(double) * (size_t)num_chunks);
    w.step_now = (long long *)(p + off);
    off += b2s_align(sizeof(long long));
    w.bytes = off;
    return w;
}

}  // namespace

extern "C" size_t b2s_optim_workspace_bytes(int num_chunks)
{
    if (num_chunks <= 0) return 0;
    return carve(nullptr, num_chunks).bytes;
}

extern "C" int b2s_optim_step(float *const *params, float *const *grads, float *const *exp_avg,
                              float *const *exp_avg_sq, int num_tensors, const int *chunks, int num_chunks,
                              const double *hyper, long long *step_dev, const b2s_optim_params *settings,
                              float *total_norm, void *workspace, size_t workspace_bytes, unsigned *status_dev,
                              void *stream_)
{
    const char *what = "b2s_optim_step";
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(num_tensors >= 1 && num_chunks >= 1, "%s: num_tensors and num_chunks must be >= 1", what);
    B2S_REQUIRE(params && grads && exp_avg && exp_avg_sq && chunks, "%s: pointer tables and chunk table required", what);
    B2S_REQUIRE((reinterpret_cast<uintptr_t>(chunks) & 15u) == 0, "%s: chunks must be 16-byte aligned", what);
    B2S_REQUIRE(hyper && step_dev && total_norm && status_dev, "%s: hyper, step_dev, total_norm and status_dev required",
                what);
    B2S_REQUIRE(settings != nullptr, "%s: settings (host) required", what);
    B2S_REQUIRE(settings->total_step >= 1, "%s: settings->total_step must be >= 1", what);
    B2S_REQUIRE(settings->decoupled == 0 || settings->decoupled == 1, "%s: settings->decoupled must be 0 or 1", what);
    B2S_REQUIRE(settings->zero_grad == 0 || settings->zero_grad == 1, "%s: settings->zero_grad must be 0 or 1", what);
    B2S_REQUIRE(settings->beta2 >= 0.0 && settings->beta2 < 1.0 && settings->eps >= 0.0 && settings->max_norm > 0.0 &&
                    settings->weight_decay >= 0.0,
                "%s: beta2 must be in [0, 1), eps and weight_decay >= 0, max_norm > 0", what);
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= b2s_optim_workspace_bytes(num_chunks),
                "%s: workspace too small", what);
    const Ws w = carve(workspace, num_chunks);
    Params q{};
    q.p = params;
    q.g = grads;
    q.m = exp_avg;
    q.v = exp_avg_sq;
    q.num_tensors = num_tensors;
    q.chunks = reinterpret_cast<const int4 *>(chunks);
    q.num_chunks = num_chunks;
    q.hyper = hyper;
    q.total_step = settings->total_step;
    q.step = step_dev;
    q.step_now = w.step_now;
    q.part = w.part;
    q.decoupled = settings->decoupled;
    q.zero_grad = settings->zero_grad;
    q.wd = (float)settings->weight_decay;
    q.beta2 = (float)settings->beta2;
    q.one_minus_beta2 = (float)(1.0 - settings->beta2);
    q.eps = (float)settings->eps;
    q.max_norm = (float)settings->max_norm;
    q.total_norm = total_norm;
    q.status = status_dev;
    k_opt_norm<<<num_chunks, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    k_opt_step<<<num_chunks, kThreads, 0, stream>>>(q);
    B2S_LAUNCH_OK();
    return 0;
}
