// pfn_train.cu -- the PointPillars feature net in training: one PFNLayer (Linear without bias, train-mode BatchNorm1d,
// ReLU, max over the T slots) forward and weight gradient without the padded [N, T, 64] map.  See include/b2second.h.
//
// Per channel c, with M = N * T slots (padded slots included, as BatchNorm1d counts them) and d_p the decorated Linear
// input of slot p (pfn_deco.cuh; 0 for padded slots):
//   mu = (1/M) sum d_p,  C = (1/M) sum (d_p - mu)(d_p - mu)^T               (float64, D x D)
//   mean_c = w_c . mu,   var_c = w_c^T C w_c,   s_c = 1 / sqrt(var_c + eps)
//   out[n, c] = max_p relu(y_p * scale_c + shift_c),  y_p = w_c . d_p,  scale_c = fp32(gamma_c s_c),
//               shift_c = fp32(beta_c - mean_c gamma_c s_c)                  (padded slots: relu(shift_c))
//   dW_c = gamma_c s_c (G - A mu - B s_c C w_c),  A = sum delta (= dbeta),  B = sum delta xhat (= dgamma),
//   G = sum delta d_p*,  over the N argmax slots p* with delta = dout[n, c] * [out[n, c] > 0], xhat = (y - mean_c) s_c.
//
// fp32 op order: the decoration of pfn_deco.cuh; y = one fmaf chain over d[0 .. D) from 0.f (the order of k_pfn);
// the BN as fmaf(y, scale_c, shift_c) and ReLU as fmaxf(., 0.f).  Everything else is float64: the moments take the
// fp32 d_p exactly, xhat = ((double)y - mean_c) * s_c.  The moments are merged Chan-style (per pillar centred on the
// pillar's mean, then pillar into warp, warp into CTA, CTA partials in order), so nothing cancels when |mu| >> std.
// Every sum runs in one fixed order (fixed grid, fixed pillar-to-warp map, no float atomics): two runs give the same
// bits.  No host sync: the entry points can be captured in a CUDA graph.
#include "bn_common.cuh"
#include "pfn_deco.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kGrid = 264;                 // moment and gradient partials: 2 CTAs per SM of an H100 SXM
constexpr int DMAX = 13;                   // F <= 8 plus the 5 offsets
constexpr int NQ = 3;                      // upper-triangle entries per lane (DMAX * (DMAX + 1) / 2 = 91 <= 96)
constexpr int PM = 112;                    // doubles per moment partial: n, mean[DMAX], q[96]
constexpr int PG = 16;                     // doubles per channel of a gradient partial: A, B, G[DMAX]
constexpr int COUT = 64;
constexpr unsigned char kPadSlot = 255;    // argmax sentinel: the maximum is the padded-slot value

inline int grid_rows(int n) { return b2s_cdiv(n, kWarps) < kGrid ? b2s_cdiv(n, kWarps) : kGrid; }

// workspace layout (bytes): moment partials, stats, gradient partials
struct Layout {
    size_t mom, mu, cov, mean, s, scale, shift, grad, total;
    explicit Layout(int n)
    {
        const size_t g = (size_t)grid_rows(n);
        mom = 0;
        mu = mom + g * PM * sizeof(double);
        cov = mu + 16 * sizeof(double);
        mean = cov + DMAX * DMAX * sizeof(double) + 8;
        s = mean + COUT * sizeof(double);
        scale = s + COUT * sizeof(double);
        shift = scale + COUT * sizeof(float);
        grad = b2s_align(shift + COUT * sizeof(float));
        total = grad + g * COUT * PG * sizeof(double);
    }
};

template <class T>
inline T *at(void *ws, size_t off) { return reinterpret_cast<T *>((char *)ws + off); }

// slot t's decorated Linear input d[0 .. D), D = NRAW + 5 (compile-time register indices)
template <int DECO>
__device__ __forceinline__ void decorated(const float *p, int F, int NRAW, const B2sPfnPillar &g, float d[DMAX])
{
    float raw[8], dec[5];
    b2s_pfn_decorate<DECO>(p, F, g, raw, dec);
#pragma unroll
    for (int k = 0; k < DMAX; ++k) {
        float v = 0.f;
        if (k < 8 && k < NRAW) v = raw[k < 8 ? k : 0];
#pragma unroll
        for (int j = 0; j < 5; ++j)
            if (k == NRAW + j) v = dec[j];
        d[k] = v;
    }
}

__device__ __forceinline__ double pick(const double v[DMAX], int k)
{
    double r = 0.0;
#pragma unroll
    for (int i = 0; i < DMAX; ++i)
        if (i == k) r = v[i];
    return r;
}

// count, mean and the lane's entries of the centred second moment of a group of rows
struct Chan {
    double n, m[DMAX], q[NQ];
};

__device__ __forceinline__ void chan_clear(Chan &a)
{
    a.n = 0.0;
#pragma unroll
    for (int k = 0; k < DMAX; ++k) a.m[k] = 0.0;
#pragma unroll
    for (int e = 0; e < NQ; ++e) a.q[e] = 0.0;
}

// a <- a merged with (nb, mb, qb) (Chan, Golub and LeVeque): q += qb + delta_i delta_j na nb / n
__device__ __forceinline__ void chan_merge(Chan &a, double nb, const double mb[DMAX], const double qb[NQ], const int ei[NQ],
                                           const int ej[NQ])
{
    if (nb == 0.0) return;
    const double n = a.n + nb, f = nb / n, h = a.n * f;
    double dl[DMAX];
#pragma unroll
    for (int k = 0; k < DMAX; ++k) dl[k] = mb[k] - a.m[k];
#pragma unroll
    for (int e = 0; e < NQ; ++e)
        if (ei[e] >= 0) a.q[e] += qb[e] + pick(dl, ei[e]) * pick(dl, ej[e]) * h;
#pragma unroll
    for (int k = 0; k < DMAX; ++k) a.m[k] += dl[k] * f;
    a.n = n;
}

// the (i, j), i <= j, of the lane's upper-triangle entries e = lane + 32 r (-1 past D (D + 1) / 2)
__device__ __forceinline__ void lane_entries(int D, int lane, int ei[NQ], int ej[NQ])
{
#pragma unroll
    for (int r = 0; r < NQ; ++r) ei[r] = ej[r] = -1;
    int e = 0;
    for (int i = 0; i < D; ++i)
        for (int j = i; j < D; ++j, ++e)
#pragma unroll
            for (int r = 0; r < NQ; ++r)
                if (e == lane + 32 * r) ei[r] = i, ej[r] = j;
}

// the CTA's warps merged in warp order into the shared state (n, m, q); each warp's state `a` is merged once
__device__ void cta_merge(const Chan &a, int D, const int ei[NQ], const int ej[NQ], double *s_n, double *s_m,
                          double *s_q)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) *s_n = 0.0;
    for (int i = threadIdx.x; i < DMAX + 96; i += blockDim.x) (i < DMAX ? s_m[i] : s_q[i - DMAX]) = 0.0;
    __syncthreads();
    for (int w = 0; w < kWarps; ++w) {
        if (warp == w) {
            Chan c;
            c.n = *s_n;
#pragma unroll
            for (int k = 0; k < DMAX; ++k) c.m[k] = s_m[k];
#pragma unroll
            for (int r = 0; r < NQ; ++r) c.q[r] = ei[r] >= 0 ? s_q[lane + 32 * r] : 0.0;
            chan_merge(c, a.n, a.m, a.q, ei, ej);
            __syncwarp();
            if (lane == 0) {
                *s_n = c.n;
#pragma unroll
                for (int k = 0; k < DMAX; ++k) s_m[k] = c.m[k];
            }
#pragma unroll
            for (int r = 0; r < NQ; ++r)
                if (ei[r] >= 0) s_q[lane + 32 * r] = c.q[r];
        }
        __syncthreads();
    }
}

// 1. moments: per-CTA (count, mean, centred second moment) of the real slots' d, in float64
template <int DECO>
__global__ void __launch_bounds__(kThreads)
k_pfn_moments(const float *__restrict__ vox, int N, int T, int F, const int *__restrict__ num,
              const int *__restrict__ coors, float vx, float vy, float xoff, float yoff, double *__restrict__ part,
              unsigned *__restrict__ status)
{
    __shared__ double s_buf[kWarps][32][DMAX + 1];
    __shared__ double s_n, s_m[DMAX], s_q[96];
    const int NRAW = DECO == B2S_PFN_RADIUS ? F - 1 : F, D = NRAW + 5;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ei[NQ], ej[NQ];
    lane_entries(D, lane, ei, ej);
    Chan acc;
    chan_clear(acc);
    for (int row = blockIdx.x * kWarps + warp; row < N; row += gridDim.x * kWarps) {
        int np = __ldg(&num[row]);
        if (np < 1 || np > T) {
            if (lane == 0 && status) atomicOr(status, B2S_STATUS_BAD_INPUT);
            np = min(max(np, 0), T);
            if (np == 0) continue;
        }
        const float *pv = vox + (size_t)row * T * F;
        const auto point = [&](int t) { return pv + (size_t)t * F; };
        const B2sPfnPillar g =
            b2s_pfn_pillar(point, np, __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4)), vx, vy, xoff, yoff);
        // the pillar's mean of d (butterfly sums: every lane ends with the same bits)
        double mp[DMAX];
#pragma unroll
        for (int k = 0; k < DMAX; ++k) mp[k] = 0.0;
        for (int t = lane; t < np; t += 32) {
            float d[DMAX];
            decorated<DECO>(point(t), F, NRAW, g, d);
#pragma unroll
            for (int k = 0; k < DMAX; ++k) mp[k] += (double)d[k];
        }
#pragma unroll
        for (int k = 0; k < DMAX; ++k) {
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) mp[k] += __shfl_xor_sync(0xffffffffu, mp[k], o);
            mp[k] /= (double)np;
        }
        // its centred second moment, 32 slots at a time through shared memory
        double qp[NQ] = {0.0, 0.0, 0.0};
        for (int t0 = 0; t0 < np; t0 += 32) {
            if (t0 + lane < np) {
                float d[DMAX];
                decorated<DECO>(point(t0 + lane), F, NRAW, g, d);
#pragma unroll
                for (int k = 0; k < DMAX; ++k) s_buf[warp][lane][k] = (double)d[k] - mp[k];
            }
            __syncwarp();
            const int cnt = min(32, np - t0);
#pragma unroll
            for (int r = 0; r < NQ; ++r)
                if (ei[r] >= 0)
                    for (int s = 0; s < cnt; ++s) qp[r] += s_buf[warp][s][ei[r]] * s_buf[warp][s][ej[r]];
            __syncwarp();
        }
        chan_merge(acc, (double)np, mp, qp, ei, ej);
    }
    cta_merge(acc, D, ei, ej, &s_n, s_m, s_q);
    double *out = part + (size_t)blockIdx.x * PM;
    for (int i = threadIdx.x; i < 1 + DMAX + 96; i += blockDim.x)
        out[i] = i == 0 ? s_n : (i <= DMAX ? s_m[i - 1] : s_q[i - 1 - DMAX]);
}

// 2. stats: the partials and the padded slots merged in one fixed order; mu, C, mean_c, s_c, the fp32 BN scale / shift
// and BatchNorm1d's running-buffer update (fp32, as torch's CUDA kernel: rm = m * mean + (1 - m) * rm, the variance
// unbiased by M / (M - 1))
__global__ void __launch_bounds__(kThreads)
k_pfn_stats(const double *__restrict__ part, int nparts, int N, int T, int D, const float *__restrict__ weight,
            const float *__restrict__ gamma, const float *__restrict__ beta, float *__restrict__ rmean,
            float *__restrict__ rvar, long long *__restrict__ nbt, float momentum, float eps, double *__restrict__ mu,
            double *__restrict__ cov, double *__restrict__ mean_c, double *__restrict__ s_c, float *__restrict__ scale,
            float *__restrict__ shift)
{
    __shared__ double s_n, s_m[DMAX], s_q[96], s_cov[DMAX * DMAX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ei[NQ], ej[NQ];
    lane_entries(D, lane, ei, ej);
    Chan acc;
    chan_clear(acc);
    for (int p = warp; p < nparts; p += kWarps) {
        const double *src = part + (size_t)p * PM;
        double mb[DMAX], qb[NQ];
#pragma unroll
        for (int k = 0; k < DMAX; ++k) mb[k] = src[1 + k];
#pragma unroll
        for (int r = 0; r < NQ; ++r) qb[r] = src[1 + DMAX + lane + 32 * r];
        chan_merge(acc, src[0], mb, qb, ei, ej);
    }
    cta_merge(acc, D, ei, ej, &s_n, s_m, s_q);
    const double M = (double)N * (double)T;
    if (warp == 0) {                  // the padded slots: M - (real slots) rows of zeros
        Chan c;
        c.n = s_n;
#pragma unroll
        for (int k = 0; k < DMAX; ++k) c.m[k] = s_m[k];
#pragma unroll
        for (int r = 0; r < NQ; ++r) c.q[r] = ei[r] >= 0 ? s_q[lane + 32 * r] : 0.0;
        const double zm[DMAX] = {}, zq[NQ] = {};
        chan_merge(c, M - c.n, zm, zq, ei, ej);
        __syncwarp();
        if (lane < D) mu[lane] = pick(c.m, lane);
        if (lane == 0)
            for (int k = 0; k < DMAX; ++k) s_m[k] = c.m[k];
#pragma unroll
        for (int r = 0; r < NQ; ++r)
            if (ei[r] >= 0) {
                const double v = c.q[r] / M;
                s_cov[ei[r] * DMAX + ej[r]] = v;
                s_cov[ej[r] * DMAX + ei[r]] = v;
            }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < DMAX * DMAX; i += blockDim.x)
        cov[i] = (i / DMAX < D && i % DMAX < D) ? s_cov[i] : 0.0;
    const int c = threadIdx.x;
    if (c < COUT) {
        const float *w = weight + (size_t)c * D;
        double m = 0.0, v = 0.0;
        for (int k = 0; k < D; ++k) {
            m += (double)w[k] * s_m[k];
            double cw = 0.0;
            for (int l = 0; l < D; ++l) cw += s_cov[k * DMAX + l] * (double)w[l];
            v += (double)w[k] * cw;
        }
        v = fmax(v, 0.0);
        const double s = b2s_bn_inv_std(v, eps);
        const double gs = (double)gamma[c] * s;
        mean_c[c] = m;
        s_c[c] = s;
        scale[c] = (float)gs;
        shift[c] = (float)((double)beta[c] - m * gs);
        b2s_bn_update_running(rmean, rvar, c, m, v, M, momentum);
        if (c == 0) *nbt += 1;
    }
}

// 3. forward: one warp per pillar, lane l owns channels l and l + 32; out = max relu(BN(y)) and the argmax slot
// (kPadSlot: the padded-slot value, taken when no real slot exceeds it)
template <int DECO>
__global__ void __launch_bounds__(kThreads)
k_pfn_train_fwd(const float *__restrict__ vox, int N, int T, int F, const int *__restrict__ num,
                const int *__restrict__ coors, const float *__restrict__ weight, const float *__restrict__ scale,
                const float *__restrict__ shift, float vx, float vy, float xoff, float yoff, float *__restrict__ out,
                unsigned char *__restrict__ arg)
{
    constexpr int NCH = COUT / 32;
    const int NRAW = DECO == B2S_PFN_RADIUS ? F - 1 : F, D = NRAW + 5;
    __shared__ float s_w[DMAX * COUT];   // [D][COUT]
    for (int i = threadIdx.x; i < D * COUT; i += blockDim.x) {
        const int c = i / D, f = i - c * D;
        s_w[f * COUT + c] = __ldg(&weight[i]);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (row >= N) return;
    const int np = min(max(__ldg(&num[row]), 0), T);
    const float *pv = vox + (size_t)row * T * F;
    const auto point = [&](int t) { return pv + (size_t)t * F; };
    const B2sPfnPillar g =
        b2s_pfn_pillar(point, np, __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4)), vx, vy, xoff, yoff);
    float sc[NCH], sh[NCH], best[NCH];
    int bi[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        sc[j] = scale[lane + 32 * j];
        sh[j] = shift[lane + 32 * j];
        best[j] = np < T ? fmaxf(sh[j], 0.f) : -INFINITY;
        bi[j] = np < T ? kPadSlot : 0;
    }
    for (int t = 0; t < np; ++t) {
        float d[DMAX];
        decorated<DECO>(point(t), F, NRAW, g, d);
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
            float y = 0.f;
#pragma unroll
            for (int k = 0; k < DMAX; ++k)
                if (k < D) y = fmaf(d[k], s_w[k * COUT + lane + 32 * j], y);
            const float v = fmaxf(fmaf(y, sc[j], sh[j]), 0.f);
            if (v > best[j]) best[j] = v, bi[j] = t;
        }
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        out[(size_t)row * COUT + lane + 32 * j] = best[j];
        arg[(size_t)row * COUT + lane + 32 * j] = (unsigned char)bi[j];
    }
}

// 4. gradient partials: per CTA and channel A = sum delta, B = sum delta xhat, G = sum delta d at the argmax slots
template <int DECO>
__global__ void __launch_bounds__(kThreads)
k_pfn_train_grad(const float *__restrict__ vox, int N, int T, int F, const int *__restrict__ num,
                 const int *__restrict__ coors, const float *__restrict__ weight, float vx, float vy, float xoff,
                 float yoff, const float *__restrict__ out, const unsigned char *__restrict__ arg,
                 const float *__restrict__ dout, const double *__restrict__ mean_c, const double *__restrict__ s_c,
                 double *__restrict__ part)
{
    constexpr int NCH = COUT / 32;
    const int NRAW = DECO == B2S_PFN_RADIUS ? F - 1 : F, D = NRAW + 5;
    __shared__ float s_w[DMAX * COUT];
    __shared__ double s_acc[COUT * PG];
    for (int i = threadIdx.x; i < D * COUT; i += blockDim.x) {
        const int c = i / D, f = i - c * D;
        s_w[f * COUT + c] = __ldg(&weight[i]);
    }
    for (int i = threadIdx.x; i < COUT * PG; i += blockDim.x) s_acc[i] = 0.0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double mc[NCH], sc[NCH], A[NCH], B[NCH], G[NCH][DMAX];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        mc[j] = mean_c[lane + 32 * j];
        sc[j] = s_c[lane + 32 * j];
        A[j] = B[j] = 0.0;
#pragma unroll
        for (int k = 0; k < DMAX; ++k) G[j][k] = 0.0;
    }
    for (int row = blockIdx.x * kWarps + warp; row < N; row += gridDim.x * kWarps) {
        const int np = min(max(__ldg(&num[row]), 0), T);
        const float *pv = vox + (size_t)row * T * F;
        const auto point = [&](int t) { return pv + (size_t)t * F; };
        const B2sPfnPillar g =
            b2s_pfn_pillar(point, np, __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4)), vx, vy, xoff, yoff);
#pragma unroll
        for (int j = 0; j < NCH; ++j) {
            const size_t o = (size_t)row * COUT + lane + 32 * j;
            if (!(__ldg(&out[o]) > 0.f)) continue;          // relu'(y) = 0 at the maximum: no gradient
            const double delta = (double)__ldg(&dout[o]);
            const int t = __ldg(&arg[o]);
            A[j] += delta;
            if (t == kPadSlot) {                             // padded slot: d = 0, xhat = -mean s
                B[j] += delta * (-mc[j] * sc[j]);
                continue;
            }
            float d[DMAX];
            decorated<DECO>(point(t), F, NRAW, g, d);
            float y = 0.f;
#pragma unroll
            for (int k = 0; k < DMAX; ++k)
                if (k < D) y = fmaf(d[k], s_w[k * COUT + lane + 32 * j], y);
            B[j] += delta * (((double)y - mc[j]) * sc[j]);
#pragma unroll
            for (int k = 0; k < DMAX; ++k) G[j][k] += delta * (double)d[k];
        }
    }
    for (int w = 0; w < kWarps; ++w) {                       // warps added in order: fixed sums
        if (warp == w) {
#pragma unroll
            for (int j = 0; j < NCH; ++j) {
                double *a = s_acc + (lane + 32 * j) * PG;
                a[0] += A[j];
                a[1] += B[j];
#pragma unroll
                for (int k = 0; k < DMAX; ++k) a[2 + k] += G[j][k];
            }
        }
        __syncthreads();
    }
    double *dst = part + (size_t)blockIdx.x * COUT * PG;
    for (int i = threadIdx.x; i < COUT * PG; i += blockDim.x) dst[i] = s_acc[i];
}

// 5. reduce: the gradient partials in CTA order; dbeta = A, dgamma = B, dW_c = gamma s (G - A mu - B s C w)
__global__ void __launch_bounds__(1024)
k_pfn_train_reduce(const double *__restrict__ part, int nparts, int D, const float *__restrict__ weight,
                   const float *__restrict__ gamma, const double *__restrict__ mu, const double *__restrict__ cov,
                   const double *__restrict__ s_c, float *__restrict__ dw, float *__restrict__ dgamma,
                   float *__restrict__ dbeta)
{
    __shared__ double s_sum[COUT * PG];
    for (int i = threadIdx.x; i < COUT * PG; i += blockDim.x) {
        double a = 0.0;
        for (int p = 0; p < nparts; ++p) a += part[(size_t)p * COUT * PG + i];
        s_sum[i] = a;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < COUT * D; i += blockDim.x) {
        const int c = i / D, k = i - c * D;
        const double *a = s_sum + c * PG;
        const double s = s_c[c];
        double cw = 0.0;
        for (int l = 0; l < D; ++l) cw += cov[k * DMAX + l] * (double)weight[c * D + l];
        dw[i] = (float)((double)gamma[c] * s * (a[2 + k] - a[0] * mu[k] - a[1] * s * cw));
        if (k == 0) {
            dgamma[c] = (float)a[1];
            dbeta[c] = (float)a[0];
        }
    }
}

int check_args(const char *who, const void *voxels, int num_rows, int max_points, int num_feat, const void *num_points,
               const void *coors, const void *weight, const void *gamma, int cout, int decoration, const void *workspace,
               size_t workspace_bytes)
{
    B2S_REQUIRE(voxels && num_points && coors && weight && gamma && workspace, "%s: a required pointer is NULL", who);
    B2S_REQUIRE(num_rows >= 1 && max_points >= 1 && max_points <= 254,
                "%s: need num_rows >= 1 and 1 <= max_points <= 254 (the argmax is one byte per channel)", who);
    B2S_REQUIRE((long long)num_rows * max_points > 1, "%s: BatchNorm1d needs more than one value per channel", who);
    B2S_REQUIRE(num_feat >= 3 && num_feat <= 8, "%s: num_feat must be 3..8", who);
    B2S_REQUIRE(cout == COUT, "%s: only Cout=64 (PillarFeatureNet num_filters=[64]) is built", who);
    B2S_REQUIRE(decoration == B2S_PFN_PLAIN || decoration == B2S_PFN_RADIUS,
                "%s: decoration must be B2S_PFN_PLAIN (0) or B2S_PFN_RADIUS (1)", who);
    B2S_REQUIRE(workspace_bytes >= Layout(num_rows).total && ((uintptr_t)workspace & 15) == 0 &&
                    ((uintptr_t)coors & 15) == 0,
                "%s: workspace smaller than b2s_pfn_train_workspace_bytes(num_rows), or workspace / coors not 16-byte "
                "aligned", who);
    return 0;
}

template <int DECO>
int forward_launch(const float *voxels, int N, int T, int F, const int *num, const int *coors, const float *weight,
                   const float *gamma, const float *beta, float *rmean, float *rvar, long long *nbt, float momentum,
                   float eps, float vx, float vy, float xoff, float yoff, float *out, unsigned char *arg, void *ws,
                   unsigned *status, cudaStream_t stream)
{
    const Layout L(N);
    const int D = (DECO == B2S_PFN_RADIUS ? F - 1 : F) + 5;
    const int gp = grid_rows(N);
    k_pfn_moments<DECO><<<gp, kThreads, 0, stream>>>(voxels, N, T, F, num, coors, vx, vy, xoff, yoff,
                                                     at<double>(ws, L.mom), status);
    B2S_LAUNCH_OK();
    k_pfn_stats<<<1, kThreads, 0, stream>>>(at<double>(ws, L.mom), gp, N, T, D, weight, gamma, beta, rmean, rvar, nbt,
                                           momentum, eps, at<double>(ws, L.mu), at<double>(ws, L.cov),
                                           at<double>(ws, L.mean), at<double>(ws, L.s), at<float>(ws, L.scale),
                                           at<float>(ws, L.shift));
    B2S_LAUNCH_OK();
    k_pfn_train_fwd<DECO><<<b2s_cdiv(N, kWarps), kThreads, 0, stream>>>(
        voxels, N, T, F, num, coors, weight, at<float>(ws, L.scale), at<float>(ws, L.shift), vx, vy, xoff, yoff, out,
        arg);
    B2S_LAUNCH_OK();
    return 0;
}

template <int DECO>
int backward_launch(const float *voxels, int N, int T, int F, const int *num, const int *coors, const float *weight,
                    const float *gamma, float vx, float vy, float xoff, float yoff, const float *out,
                    const unsigned char *arg, const float *dout, void *ws, float *dw, float *dgamma, float *dbeta,
                    cudaStream_t stream)
{
    const Layout L(N);
    const int D = (DECO == B2S_PFN_RADIUS ? F - 1 : F) + 5;
    const int gp = grid_rows(N);
    k_pfn_train_grad<DECO><<<gp, kThreads, 0, stream>>>(voxels, N, T, F, num, coors, weight, vx, vy, xoff, yoff, out,
                                                        arg, dout, at<double>(ws, L.mean), at<double>(ws, L.s),
                                                        at<double>(ws, L.grad));
    B2S_LAUNCH_OK();
    k_pfn_train_reduce<<<1, 1024, 0, stream>>>(at<double>(ws, L.grad), gp, D, weight, gamma, at<double>(ws, L.mu),
                                               at<double>(ws, L.cov), at<double>(ws, L.s), dw, dgamma, dbeta);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

extern "C" size_t b2s_pfn_train_workspace_bytes(int num_rows) { return num_rows < 1 ? 0 : Layout(num_rows).total; }

extern "C" int b2s_pfn_train_forward(const float *voxels, int num_rows, int max_points, int num_feat,
                                     const int *num_points, const int *coors, const float *weight, const float *gamma,
                                     const float *beta, int cout, float *running_mean, float *running_var,
                                     int64_t *num_batches_tracked, float momentum, float eps, float vx, float vy,
                                     float x_offset, float y_offset, int decoration, float *out, uint8_t *argmax,
                                     void *workspace, size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    const char *who = "b2s_pfn_train_forward";
    if (int rc = check_args(who, voxels, num_rows, max_points, num_feat, num_points, coors, weight, gamma, cout,
                            decoration, workspace, workspace_bytes))
        return rc;
    B2S_REQUIRE(beta && running_mean && running_var && num_batches_tracked && out && argmax,
                "%s: a required pointer is NULL", who);
    B2S_REQUIRE(eps > 0.f && momentum >= 0.f && momentum <= 1.f, "%s: need eps > 0 and 0 <= momentum <= 1", who);
    cudaStream_t stream = (cudaStream_t)stream_;
    long long *nbt = reinterpret_cast<long long *>(num_batches_tracked);
    if (decoration == B2S_PFN_RADIUS)
        return forward_launch<B2S_PFN_RADIUS>(voxels, num_rows, max_points, num_feat, num_points, coors, weight, gamma,
                                              beta, running_mean, running_var, nbt, momentum, eps, vx, vy, x_offset,
                                              y_offset, out, argmax, workspace, status_dev, stream);
    return forward_launch<B2S_PFN_PLAIN>(voxels, num_rows, max_points, num_feat, num_points, coors, weight, gamma, beta,
                                         running_mean, running_var, nbt, momentum, eps, vx, vy, x_offset, y_offset, out,
                                         argmax, workspace, status_dev, stream);
}

extern "C" int b2s_pfn_train_backward(const float *voxels, int num_rows, int max_points, int num_feat,
                                      const int *num_points, const int *coors, const float *weight, const float *gamma,
                                      int cout, float vx, float vy, float x_offset, float y_offset, int decoration,
                                      const float *out, const uint8_t *argmax, const float *dout, void *workspace,
                                      size_t workspace_bytes, float *dweight, float *dgamma, float *dbeta,
                                      void *stream_)
{
    const char *who = "b2s_pfn_train_backward";
    if (int rc = check_args(who, voxels, num_rows, max_points, num_feat, num_points, coors, weight, gamma, cout,
                            decoration, workspace, workspace_bytes))
        return rc;
    B2S_REQUIRE(out && argmax && dout && dweight && dgamma && dbeta, "%s: a required pointer is NULL", who);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (decoration == B2S_PFN_RADIUS)
        return backward_launch<B2S_PFN_RADIUS>(voxels, num_rows, max_points, num_feat, num_points, coors, weight, gamma,
                                               vx, vy, x_offset, y_offset, out, argmax, dout, workspace, dweight,
                                               dgamma, dbeta, stream);
    return backward_launch<B2S_PFN_PLAIN>(voxels, num_rows, max_points, num_feat, num_points, coors, weight, gamma, vx,
                                          vy, x_offset, y_offset, out, argmax, dout, workspace, dweight, dgamma, dbeta,
                                          stream);
}
