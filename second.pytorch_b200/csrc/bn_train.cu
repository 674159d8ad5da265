// bn_train.cu -- BatchNorm (1d or 2d) followed by ReLU in training mode, forward and backward, on an fp32 tensor with C
// channels in one of two layouts (see include/b2second.h):
//   B2S_LAYOUT_NHWC  rows [M, C]: BatchNorm1d input, or a channels_last NCHW map viewed as [B*H*W, C];
//   B2S_LAYOUT_NCHW  [B, C, HW] contiguous, M = B * HW.
//
// Per channel c, with K_c = the channel's first element (a shift taken from the data):
//   S1 = sum (x - K), S2 = sum (x - K)^2                 (float64, per-CTA partials added in one fixed order)
//   mean = K + S1 / M,  var = S2 / M - (S1 / M)^2,  s = 1 / sqrt(var + eps)          (float64; var < 0 -> 0)
//   y = relu(v),  v = fmaf(x - mu32, a32, beta)   with mu32 = fp32(mean), a32 = fp32(gamma s)
// Because K is one of the channel's own values, |mean - K| is of the order of the spread, so S2 / M - (S1 / M)^2 does
// not cancel when |mean| >> std (it would with sum x^2 - M mean^2).  The apply form subtracts the fp32 mean first, so
// it does not cancel either; tests/bn_train_ref.py states its per-element bound.
// Backward, with the mask recomputed from x by the forward's own expression (nothing but x and the workspace is kept):
//   g = [v > 0 or v is NaN] dY  (torch's ReLU backward: threshold_backward(dY, y, 0) passes where !(y <= 0))
//   dbeta = sum g,  dgamma = sum g xhat,  xhat = ((double)x - mean) s     (float64 partials in one fixed order)
//   dX = fp32(gamma s (g - dbeta / M - xhat dgamma / M))                   (float64 per element)
// No float atomics: two runs give the same bits.  No host value is read and nothing syncs, so both directions can be
// captured in a CUDA graph.
#include "bn_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kGrid = 396;                 // sum partials: 3 CTAs per SM of an H100 SXM (80 registers)
constexpr int kApplyGrid = 132 * 8;        // grid-stride elementwise passes
constexpr int kMaxC = 1024;                // one finalize thread per channel
enum { STATS = 0, GRAD = 1 };

// the number of CTAs (= partials) of a sum pass
inline int num_parts(int layout, long long M, int C, int HW)
{
    if (layout == B2S_LAYOUT_NHWC) {
        const int rpp = kThreads / (C / 4);
        return (int)std::min<long long>(kGrid, (M + rpp - 1) / rpp);
    }
    const long long per_chunk = 4LL * kThreads;            // at least 4 elements per thread
    return (int)std::max<long long>(1, std::min<long long>((kGrid + C - 1) / C, (M + per_chunk - 1) / per_chunk));
}

// workspace layout (bytes): the forward's and the backward's sum partials [parts][2][C] (double), then per channel
// mean, s (double), mu32, a32, b32 (float) and the backward's coefficients gamma s, dbeta / M, dgamma / M (double)
struct Layout {
    size_t fwd, bwd, mean, s, mu32, a32, b32, coef, total;
    Layout(int layout, long long M, int C, int HW)
    {
        const size_t part = (size_t)num_parts(layout, M, C, HW) * 2 * C * sizeof(double);
        fwd = 0;
        bwd = b2s_align(fwd + part);
        mean = b2s_align(bwd + part);
        s = b2s_align(mean + C * sizeof(double));
        mu32 = b2s_align(s + C * sizeof(double));
        a32 = b2s_align(mu32 + C * sizeof(float));
        b32 = b2s_align(a32 + C * sizeof(float));
        coef = b2s_align(b32 + C * sizeof(float));
        total = b2s_align(coef + 3 * C * sizeof(double));
    }
};

template <class T>
inline T *at(void *ws, size_t off) { return reinterpret_cast<T *>((char *)ws + off); }

struct Stats {                             // the per-channel values the passes after the forward's finalize read
    const double *mean, *s;
    const float *mu32, *a32, *b32;
};

inline Stats stats_of(void *ws, const Layout &L)
{
    return {at<double>(ws, L.mean), at<double>(ws, L.s), at<float>(ws, L.mu32), at<float>(ws, L.a32),
            at<float>(ws, L.b32)};
}

// BN before the ReLU, in fp32: the apply pass and the backward's mask both call this, so they see the same bits
__device__ __forceinline__ float bn_pre(float x, float mu, float a, float b) { return __fmaf_rn(__fsub_rn(x, mu), a, b); }
__device__ __forceinline__ float relu(float v) { return v <= 0.f ? 0.f : v; }     // NaN passes, as in torch

// one element's contribution to the channel's two sums
template <int MODE>
__device__ __forceinline__ void accumulate(float x, float dy, double K, double mean, double s, float mu, float a,
                                           float b, double &s1, double &s2)
{
    if (MODE == STATS) {
        const double d = (double)x - K;
        s1 += d;
        s2 = fma(d, d, s2);
    } else {
        if (bn_pre(x, mu, a, b) <= 0.f) return;
        const double g = (double)dy;
        s1 += g;
        s2 = fma(g, ((double)x - mean) * s, s2);
    }
}

__device__ __forceinline__ float get(const float4 &v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }

// 1a. sum partials, rows: thread t owns channels 4 q .. 4 q + 3 (q = t % Q, Q = C / 4) of rows r0, r0 + rpp, ...
// (r0 = t / Q, rpp = 256 / Q rows per CTA step); the rpp row groups are added in order through shared memory
template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_bn_sums_rows(const float *__restrict__ x, const float *__restrict__ dy, long long M, int C, Stats st,
               double *__restrict__ part)
{
    __shared__ double s_red[kThreads][8];
    const int Q = C / 4, rpp = kThreads / Q;
    const int q = threadIdx.x % Q, r0 = threadIdx.x / Q;
    double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
    if (r0 < rpp) {
        double K[4] = {}, mean[4] = {}, s[4] = {};
        float4 mu = {}, a = {}, b = {};
        if (MODE == STATS) {
            const float4 k = __ldg(reinterpret_cast<const float4 *>(x) + q);
#pragma unroll
            for (int j = 0; j < 4; ++j) K[j] = (double)get(k, j);
        } else {
            mu = reinterpret_cast<const float4 *>(st.mu32)[q];
            a = reinterpret_cast<const float4 *>(st.a32)[q];
            b = reinterpret_cast<const float4 *>(st.b32)[q];
#pragma unroll
            for (int j = 0; j < 4; ++j) mean[j] = st.mean[4 * q + j], s[j] = st.s[4 * q + j];
        }
        const long long step = (long long)gridDim.x * rpp;
        for (long long row = (long long)blockIdx.x * rpp + r0; row < M; row += 2 * step) {
            const bool two = row + step < M;                  // two independent loads in flight
            const float4 *xp = reinterpret_cast<const float4 *>(x + row * C) + q;
            const float4 x0 = __ldg(xp), x1 = two ? __ldg(xp + step * Q) : x0;
            float4 g0 = {}, g1 = {};
            if (MODE == GRAD) {
                const float4 *gp = reinterpret_cast<const float4 *>(dy + row * C) + q;
                g0 = __ldg(gp), g1 = two ? __ldg(gp + step * Q) : g0;
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
                accumulate<MODE>(get(x0, j), get(g0, j), K[j], mean[j], s[j], get(mu, j), get(a, j), get(b, j), s1[j],
                                 s2[j]);
            if (two)
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    accumulate<MODE>(get(x1, j), get(g1, j), K[j], mean[j], s[j], get(mu, j), get(a, j), get(b, j),
                                     s1[j], s2[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) s_red[threadIdx.x][j] = s1[j], s_red[threadIdx.x][4 + j] = s2[j];
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double t1 = 0.0, t2 = 0.0;
        for (int r = 0; r < rpp; ++r) {
            t1 += s_red[r * Q + c / 4][c % 4];
            t2 += s_red[r * Q + c / 4][4 + c % 4];
        }
        part[(size_t)blockIdx.x * 2 * C + c] = t1;
        part[(size_t)blockIdx.x * 2 * C + C + c] = t2;
    }
}

// 1b. sum partials, NCHW: CTA (k, c) sums channel c's elements j in chunk k of [0, M), element j at
// x[(j / HW) * C * HW + c * HW + j % HW]; warp butterflies, then the warps in order
template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_bn_sums_nchw(const float *__restrict__ x, const float *__restrict__ dy, long long M, int C, int HW, Stats st,
               double *__restrict__ part)
{
    __shared__ double s_w[kThreads / 32][2];
    const int c = blockIdx.y, nck = gridDim.x;
    const long long chunk = (M + nck - 1) / nck, j0 = blockIdx.x * chunk, j1 = min(M, j0 + chunk);
    double K = 0.0, mean = 0.0, s = 0.0;
    float mu = 0.f, a = 0.f, b = 0.f;
    if (MODE == STATS) {
        K = (double)__ldg(&x[(size_t)c * HW]);
    } else {
        mean = st.mean[c], s = st.s[c], mu = st.mu32[c], a = st.a32[c], b = st.b32[c];
    }
    double s1 = 0.0, s2 = 0.0;
    constexpr int U = 4;
    for (long long j = j0 + threadIdx.x; j < j1; j += U * kThreads) {
        float xv[U], gv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long e = j + u * kThreads;
            xv[u] = gv[u] = 0.f;
            if (e < j1) {
                const size_t o = (size_t)(e / HW) * C * HW + (size_t)c * HW + (size_t)(e % HW);
                xv[u] = __ldg(&x[o]);
                if (MODE == GRAD) gv[u] = __ldg(&dy[o]);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (j + u * kThreads < j1) accumulate<MODE>(xv[u], gv[u], K, mean, s, mu, a, b, s1, s2);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_w[warp][0] = s1, s_w[warp][1] = s2;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t1 = 0.0, t2 = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) t1 += s_w[w][0], t2 += s_w[w][1];
        part[(size_t)blockIdx.x * 2 * C + c] = t1;
        part[(size_t)blockIdx.x * 2 * C + C + c] = t2;
    }
}

// the two sums of channel c = threadIdx.x (< C) over all partials, in one fixed order: the kMaxC / C threads of a
// channel each add every (kMaxC / C)-th partial in order, then their sums are added in thread order
__device__ void sum_partials(const double *__restrict__ part, int nparts, int C, double &t1, double &t2)
{
    __shared__ double s_sub[kMaxC][2];
    const int S = kMaxC / C, c = threadIdx.x % C, k = threadIdx.x / C;
    double a1 = 0.0, a2 = 0.0;
    if (k < S)
        for (int p = k; p < nparts; p += S) {
            a1 += part[(size_t)p * 2 * C + c];
            a2 += part[(size_t)p * 2 * C + C + c];
        }
    s_sub[threadIdx.x][0] = a1;
    s_sub[threadIdx.x][1] = a2;
    __syncthreads();
    t1 = t2 = 0.0;
    if (threadIdx.x < C)
        for (int i = 0; i < S; ++i) t1 += s_sub[i * C + c][0], t2 += s_sub[i * C + c][1];
}

// 2. forward finalize (one CTA): mean, var, s, the fp32 apply factors and the running-buffer update
__global__ void __launch_bounds__(kMaxC)
k_bn_finalize_fwd(const double *__restrict__ part, int nparts, const float *__restrict__ x, int layout, long long M,
                  int C, int HW, const float *__restrict__ gamma, const float *__restrict__ beta,
                  float *__restrict__ rmean, float *__restrict__ rvar, long long *__restrict__ nbt, float momentum,
                  float eps, double *__restrict__ mean_o, double *__restrict__ s_o, float *__restrict__ mu32,
                  float *__restrict__ a32, float *__restrict__ b32)
{
    double S1, S2;
    sum_partials(part, nparts, C, S1, S2);
    const int c = threadIdx.x;
    if (c >= C) return;
    const double Md = (double)M;
    const double K = (double)x[layout == B2S_LAYOUT_NHWC ? (size_t)c : (size_t)c * HW];
    const double m1 = S1 / Md, mean = K + m1;
    double var = S2 / Md - m1 * m1;
    var = var < 0.0 ? 0.0 : var;                             // rounding only; NaN stays NaN
    const double s = b2s_bn_inv_std(var, eps);
    mean_o[c] = mean;
    s_o[c] = s;
    mu32[c] = (float)mean;
    a32[c] = (float)((double)gamma[c] * s);
    b32[c] = beta[c];
    b2s_bn_update_running(rmean, rvar, c, mean, var, Md, momentum);
    if (c == 0) *nbt += 1;
}

// 3. apply: y = relu(bn_pre(x)) in x's layout; VEC: four consecutive elements per thread (rows always; NCHW when
// HW % 4 == 0 and the pointers are 16-byte aligned)
template <int LAYOUT, bool VEC>
__global__ void __launch_bounds__(kThreads)
k_bn_apply(const float *__restrict__ x, long long n, int C, int HW, Stats st, float *__restrict__ y)
{
    const long long stride = (long long)gridDim.x * blockDim.x;
    if (VEC) {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n / 4; i += stride) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(x) + i);
            float4 o;
            if (LAYOUT == B2S_LAYOUT_NHWC) {
                const int q = (int)(i % (C / 4));
                const float4 mu = reinterpret_cast<const float4 *>(st.mu32)[q];
                const float4 a = reinterpret_cast<const float4 *>(st.a32)[q];
                const float4 b = reinterpret_cast<const float4 *>(st.b32)[q];
                o = {relu(bn_pre(v.x, mu.x, a.x, b.x)), relu(bn_pre(v.y, mu.y, a.y, b.y)),
                     relu(bn_pre(v.z, mu.z, a.z, b.z)), relu(bn_pre(v.w, mu.w, a.w, b.w))};
            } else {
                const int c = (int)((4 * i / HW) % C);
                const float mu = st.mu32[c], a = st.a32[c], b = st.b32[c];
                o = {relu(bn_pre(v.x, mu, a, b)), relu(bn_pre(v.y, mu, a, b)), relu(bn_pre(v.z, mu, a, b)),
                     relu(bn_pre(v.w, mu, a, b))};
            }
            reinterpret_cast<float4 *>(y)[i] = o;
        }
    } else {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
            const int c = LAYOUT == B2S_LAYOUT_NHWC ? (int)(i % C) : (int)((i / HW) % C);
            y[i] = relu(bn_pre(__ldg(&x[i]), st.mu32[c], st.a32[c], st.b32[c]));
        }
    }
}

// 4. backward finalize (one CTA): dgamma, dbeta and the dX coefficients gamma s, dbeta / M, dgamma / M
__global__ void __launch_bounds__(kMaxC)
k_bn_finalize_bwd(const double *__restrict__ part, int nparts, long long M, int C, const float *__restrict__ gamma,
                  const double *__restrict__ s_c, float *__restrict__ dgamma, float *__restrict__ dbeta,
                  double *__restrict__ coef)
{
    double db, dg;
    sum_partials(part, nparts, C, db, dg);
    const int c = threadIdx.x;
    if (c >= C) return;
    dbeta[c] = (float)db;
    dgamma[c] = (float)dg;
    coef[c] = (double)gamma[c] * s_c[c];
    coef[C + c] = db / (double)M;
    coef[2 * C + c] = dg / (double)M;
}

__device__ __forceinline__ float dx_of(float x, float dy, int c, const Stats &st, const double *__restrict__ coef, int C)
{
    const float v = bn_pre(x, st.mu32[c], st.a32[c], st.b32[c]);
    const double g = v <= 0.f ? 0.0 : (double)dy;
    const double xh = ((double)x - st.mean[c]) * st.s[c];
    return (float)(coef[c] * ((g - coef[C + c]) - xh * coef[2 * C + c]));
}

// 5. dX = gamma s (g - dbeta / M - xhat dgamma / M) in x's layout
template <int LAYOUT, bool VEC>
__global__ void __launch_bounds__(kThreads)
k_bn_dx(const float *__restrict__ x, const float *__restrict__ dy, long long n, int C, int HW, Stats st,
        const double *__restrict__ coef, float *__restrict__ dx)
{
    const long long stride = (long long)gridDim.x * blockDim.x;
    if (VEC) {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n / 4; i += stride) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(x) + i);
            const float4 g = __ldg(reinterpret_cast<const float4 *>(dy) + i);
            float4 o;
            if (LAYOUT == B2S_LAYOUT_NHWC) {
                const int c = (int)(i % (C / 4)) * 4;
                o = {dx_of(v.x, g.x, c, st, coef, C), dx_of(v.y, g.y, c + 1, st, coef, C),
                     dx_of(v.z, g.z, c + 2, st, coef, C), dx_of(v.w, g.w, c + 3, st, coef, C)};
            } else {
                const int c = (int)((4 * i / HW) % C);
                o = {dx_of(v.x, g.x, c, st, coef, C), dx_of(v.y, g.y, c, st, coef, C), dx_of(v.z, g.z, c, st, coef, C),
                     dx_of(v.w, g.w, c, st, coef, C)};
            }
            reinterpret_cast<float4 *>(dx)[i] = o;
        }
    } else {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
            const int c = LAYOUT == B2S_LAYOUT_NHWC ? (int)(i % C) : (int)((i / HW) % C);
            dx[i] = dx_of(__ldg(&x[i]), __ldg(&dy[i]), c, st, coef, C);
        }
    }
}

inline bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

int check_args(const char *who, int layout, int batch, int channels, int spatial, const void *x, const void *gamma,
               const void *workspace, size_t workspace_bytes)
{
    B2S_REQUIRE(x && gamma && workspace, "%s: a required pointer is NULL", who);
    B2S_REQUIRE(layout == B2S_LAYOUT_NCHW || layout == B2S_LAYOUT_NHWC,
                "%s: layout must be B2S_LAYOUT_NCHW (0) or B2S_LAYOUT_NHWC (1, rows [M, C])", who);
    B2S_REQUIRE(batch >= 1 && spatial >= 1, "%s: need batch >= 1 and spatial >= 1", who);
    B2S_REQUIRE((long long)batch * spatial >= 2, "%s: BatchNorm needs more than one value per channel (M >= 2)", who);
    B2S_REQUIRE(channels >= 4 && channels <= kMaxC && channels % 4 == 0,
                "%s: channels must be a multiple of 4 in 4..1024", who);
    B2S_REQUIRE(workspace_bytes >= Layout(layout, (long long)batch * spatial, channels, spatial).total &&
                    aligned16(workspace),
                "%s: workspace smaller than b2s_bn_relu_train_workspace_bytes(...) or not 16-byte aligned", who);
    return 0;
}

template <int LAYOUT, bool VEC>
void launch_apply(const float *x, long long n, int C, int HW, const Stats &st, float *y, cudaStream_t stream)
{
    const long long work = VEC ? n / 4 : n;
    const int grid = (int)std::min<long long>(kApplyGrid, (work + kThreads - 1) / kThreads);
    k_bn_apply<LAYOUT, VEC><<<grid, kThreads, 0, stream>>>(x, n, C, HW, st, y);
}

template <int LAYOUT, bool VEC>
void launch_dx(const float *x, const float *dy, long long n, int C, int HW, const Stats &st, const double *coef,
               float *dx, cudaStream_t stream)
{
    const long long work = VEC ? n / 4 : n;
    const int grid = (int)std::min<long long>(kApplyGrid, (work + kThreads - 1) / kThreads);
    k_bn_dx<LAYOUT, VEC><<<grid, kThreads, 0, stream>>>(x, dy, n, C, HW, st, coef, dx);
}

template <int MODE>
void launch_sums(const float *x, const float *dy, int layout, long long M, int C, int HW, const Stats &st,
                 double *part, cudaStream_t stream)
{
    const int np = num_parts(layout, M, C, HW);
    if (layout == B2S_LAYOUT_NHWC)
        k_bn_sums_rows<MODE><<<np, kThreads, 0, stream>>>(x, dy, M, C, st, part);
    else
        k_bn_sums_nchw<MODE><<<dim3(np, C), kThreads, 0, stream>>>(x, dy, M, C, HW, st, part);
}

}  // namespace

extern "C" size_t b2s_bn_relu_train_workspace_bytes(int layout, int batch, int channels, int spatial)
{
    if ((layout != B2S_LAYOUT_NCHW && layout != B2S_LAYOUT_NHWC) || batch < 1 || spatial < 1 || channels < 4 ||
        channels > kMaxC || channels % 4)
        return 0;
    return Layout(layout, (long long)batch * spatial, channels, spatial).total;
}

extern "C" int b2s_bn_relu_train_forward(const float *x, int layout, int batch, int channels, int spatial,
                                         const float *gamma, const float *beta, float *running_mean,
                                         float *running_var, int64_t *num_batches_tracked, float momentum, float eps,
                                         float *y, void *workspace, size_t workspace_bytes, void *stream_)
{
    const char *who = "b2s_bn_relu_train_forward";
    if (int rc = check_args(who, layout, batch, channels, spatial, x, gamma, workspace, workspace_bytes)) return rc;
    B2S_REQUIRE(beta && running_mean && running_var && num_batches_tracked && y, "%s: a required pointer is NULL", who);
    B2S_REQUIRE(layout == B2S_LAYOUT_NCHW || (aligned16(x) && aligned16(y)), "%s: rows must be 16-byte aligned", who);
    B2S_REQUIRE(eps > 0.f && momentum >= 0.f && momentum <= 1.f, "%s: need eps > 0 and 0 <= momentum <= 1", who);
    cudaStream_t stream = (cudaStream_t)stream_;
    const long long M = (long long)batch * spatial, n = M * channels;
    const int C = channels, HW = layout == B2S_LAYOUT_NHWC ? 1 : spatial;
    const Layout L(layout, M, C, spatial);
    const Stats st = stats_of(workspace, L);
    launch_sums<STATS>(x, nullptr, layout, M, C, HW, st, at<double>(workspace, L.fwd), stream);
    B2S_LAUNCH_OK();
    k_bn_finalize_fwd<<<1, kMaxC, 0, stream>>>(at<double>(workspace, L.fwd), num_parts(layout, M, C, spatial), x,
                                               layout, M, C, HW, gamma, beta, running_mean, running_var,
                                               reinterpret_cast<long long *>(num_batches_tracked), momentum, eps,
                                               at<double>(workspace, L.mean), at<double>(workspace, L.s),
                                               at<float>(workspace, L.mu32), at<float>(workspace, L.a32),
                                               at<float>(workspace, L.b32));
    B2S_LAUNCH_OK();
    if (layout == B2S_LAYOUT_NHWC)
        launch_apply<B2S_LAYOUT_NHWC, true>(x, n, C, HW, st, y, stream);
    else if (HW % 4 == 0 && aligned16(x) && aligned16(y))
        launch_apply<B2S_LAYOUT_NCHW, true>(x, n, C, HW, st, y, stream);
    else
        launch_apply<B2S_LAYOUT_NCHW, false>(x, n, C, HW, st, y, stream);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_bn_relu_train_backward(const float *x, const float *dy, int layout, int batch, int channels,
                                          int spatial, const float *gamma, void *workspace, size_t workspace_bytes,
                                          float *dx, float *dgamma, float *dbeta, void *stream_)
{
    const char *who = "b2s_bn_relu_train_backward";
    if (int rc = check_args(who, layout, batch, channels, spatial, x, gamma, workspace, workspace_bytes)) return rc;
    B2S_REQUIRE(dy && dgamma && dbeta, "%s: a required pointer is NULL", who);
    B2S_REQUIRE(layout == B2S_LAYOUT_NCHW || (aligned16(x) && aligned16(dy) && (!dx || aligned16(dx))),
                "%s: rows must be 16-byte aligned", who);
    cudaStream_t stream = (cudaStream_t)stream_;
    const long long M = (long long)batch * spatial, n = M * channels;
    const int C = channels, HW = layout == B2S_LAYOUT_NHWC ? 1 : spatial;
    const Layout L(layout, M, C, spatial);
    const Stats st = stats_of(workspace, L);
    launch_sums<GRAD>(x, dy, layout, M, C, HW, st, at<double>(workspace, L.bwd), stream);
    B2S_LAUNCH_OK();
    k_bn_finalize_bwd<<<1, kMaxC, 0, stream>>>(at<double>(workspace, L.bwd), num_parts(layout, M, C, spatial), M, C,
                                               gamma, st.s, dgamma, dbeta, at<double>(workspace, L.coef));
    B2S_LAUNCH_OK();
    if (!dx) return 0;
    const double *coef = at<double>(workspace, L.coef);
    if (layout == B2S_LAYOUT_NHWC)
        launch_dx<B2S_LAYOUT_NHWC, true>(x, dy, n, C, HW, st, coef, dx, stream);
    else if (HW % 4 == 0 && aligned16(x) && aligned16(dy) && aligned16(dx))
        launch_dx<B2S_LAYOUT_NCHW, true>(x, dy, n, C, HW, st, coef, dx, stream);
    else
        launch_dx<B2S_LAYOUT_NCHW, false>(x, dy, n, C, HW, st, coef, dx, stream);
    B2S_LAUNCH_OK();
    return 0;
}
