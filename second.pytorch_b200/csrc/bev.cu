// bev.cu -- sparse rows -> dense BEV map (b2s_to_bev) and the PointPillars feature net (b2s_pfn).
// See include/b2second.h.  Pure HBM-bound data movement: zero-fill the dense map once, then one
// scattered write per (row, channel).
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBlocks = 132 * 8;   // bounded grids + grid-stride loops: cost follows the live row count

inline int bounded_grid(long long items)
{
    long long b = (items + kThreads - 1) / kThreads;
    if (b < 1) b = 1;
    return (int)(b < kMaxBlocks ? b : kMaxBlocks);
}

__global__ void k_to_bev(const float *__restrict__ feat, const int *__restrict__ coors,
                         const int *__restrict__ n_dev, int cap_rows, int C, int batch, int D, int H, int W,
                         float *__restrict__ out, int layout)
{
    const int n = min(*n_dev, cap_rows);
    const long long total = (long long)n * C;
    for (long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x; gid < total;
         gid += (long long)gridDim.x * blockDim.x) {
        int row = (int)(gid / C), c = (int)(gid % C);
        int4 q = __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4));  // b,z,y,x
        if ((unsigned)q.x >= (unsigned)batch || (unsigned)q.y >= (unsigned)D || (unsigned)q.z >= (unsigned)H ||
            (unsigned)q.w >= (unsigned)W)
            continue;
        float v = __ldg(&feat[gid]);
        size_t CD = (size_t)C * D;
        size_t ch = (size_t)c * D + q.y;
        size_t idx;
        if (layout == B2S_LAYOUT_NCHW) idx = (((size_t)q.x * CD + ch) * H + q.z) * W + q.w;
        else idx = (((size_t)q.x * H + q.z) * W + q.w) * CD + ch;
        out[idx] = v;
    }
}

// tensor-core RPN input: NHWC + one-pixel zero halo, fp16 hi/lo planes (3xF16 split).  The rows come either as fp32
// (PointPillars: the PFN output) or already split (the last sparse layer's hi/lo planes, row stride feat_stride halves).
__global__ void k_to_bev_tc(const float *__restrict__ feat, const __half *__restrict__ feat_hi,
                            const __half *__restrict__ feat_lo, int feat_stride, const int *__restrict__ coors,
                            const int *__restrict__ n_dev, int cap_rows, int C, int batch, int D, int H, int W,
                            __half *__restrict__ out_hi, __half *__restrict__ out_lo, uint8_t *__restrict__ occ)
{
    const int n = min(*n_dev, cap_rows);
    const long long total = (long long)n * C;
    for (long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x; gid < total;
         gid += (long long)gridDim.x * blockDim.x) {
        int row = (int)(gid / C), c = (int)(gid % C);
        int4 q = __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4));  // b,z,y,x
        if ((unsigned)q.x >= (unsigned)batch || (unsigned)q.y >= (unsigned)D || (unsigned)q.z >= (unsigned)H ||
            (unsigned)q.w >= (unsigned)W)
            continue;
        size_t CD = (size_t)C * D;
        size_t idx = (((size_t)q.x * (H + 2) + (q.z + 1)) * (W + 2) + (q.w + 1)) * CD + (size_t)c * D + q.y;
        if (occ && c == 0) occ[((size_t)q.x * H + q.z) * W + q.w] = 1;      // the pixel holds data (b2s_rpn_bg_plan)
        if (feat) {
            const uint32_t pk = b2s_tc::split_f16(__ldg(&feat[gid]));
            out_hi[idx] = __ushort_as_half((unsigned short)(pk & 0xFFFFu));
            out_lo[idx] = __ushort_as_half((unsigned short)(pk >> 16));
        } else {
            out_hi[idx] = feat_hi[(size_t)row * feat_stride + c];
            out_lo[idx] = feat_lo[(size_t)row * feat_stride + c];
        }
    }
}

// PointPillars PFN (single layer): one warp per pillar; lane l owns output channels l, l+32, ...
// decorate each point with (xyz - mean xyz) and (xy - pillar centre), Linear(F+5 -> COUT), BN, ReLU,
// max over the T slots (padded slots contribute relu(shift), exactly like the masked zero rows upstream).
template <int COUT>
__global__ void __launch_bounds__(kThreads)
k_pfn(const float *__restrict__ points, int F, const int *__restrict__ slots, const int *__restrict__ num,
      const int *__restrict__ coors, const int *__restrict__ n_dev, int cap_rows, int T,
      const float *__restrict__ weight, const float *__restrict__ scale, const float *__restrict__ shift,
      float vx, float vy, float xoff, float yoff, float *__restrict__ out)
{
    constexpr int NCH = COUT / 32;
    const int FIN = F + 5;
    extern __shared__ float s_w[];  // [FIN][COUT] transposed weights
    for (int i = threadIdx.x; i < FIN * COUT; i += blockDim.x) {
        int c = i / FIN, f = i - c * FIN;  // weight is [COUT][FIN]
        s_w[f * COUT + c] = __ldg(&weight[i]);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int n = min(*n_dev, cap_rows);
    if (warp >= n) return;
    const int row = warp;
    const int np = num[row];
    const int *sl = slots + (size_t)row * T;
    // mean of xyz over the valid points, summed in slot order (sequential fp32 like the oracle)
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int t = 0; t < np; ++t) {
        const float *p = points + (size_t)__ldg(&sl[t]) * F;
        sx = __fadd_rn(sx, __ldg(&p[0]));
        sy = __fadd_rn(sy, __ldg(&p[1]));
        sz = __fadd_rn(sz, __ldg(&p[2]));
    }
    const float fn = (float)np;
    const float mx = __fdiv_rn(sx, fn), my = __fdiv_rn(sy, fn), mz = __fdiv_rn(sz, fn);
    int4 q = __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4));
    const float cx = __fadd_rn(__fmul_rn((float)q.w, vx), xoff);
    const float cy = __fadd_rn(__fmul_rn((float)q.z, vy), yoff);
    float sc[NCH], sh[NCH], best[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        sc[j] = __ldg(&scale[lane + 32 * j]);
        sh[j] = __ldg(&shift[lane + 32 * j]);
        // padded slots are all-zero rows upstream: linear -> 0, BN -> shift, ReLU
        best[j] = (np < T) ? fmaxf(sh[j], 0.f) : -INFINITY;
    }
    for (int t = 0; t < np; ++t) {
        const float *p = points + (size_t)__ldg(&sl[t]) * F;
        float feat[16];
#pragma unroll
        for (int f = 0; f < 8; ++f) feat[f] = (f < F) ? __ldg(&p[f]) : 0.f;
        float acc[NCH];
#pragma unroll
        for (int j = 0; j < NCH; ++j) acc[j] = 0.f;
        for (int f = 0; f < F; ++f)
#pragma unroll
            for (int j = 0; j < NCH; ++j) acc[j] = fmaf(feat[f], s_w[f * COUT + lane + 32 * j], acc[j]);
        float dec[5] = {__fsub_rn(feat[0], mx), __fsub_rn(feat[1], my), __fsub_rn(feat[2], mz),
                        __fsub_rn(feat[0], cx), __fsub_rn(feat[1], cy)};
#pragma unroll
        for (int f = 0; f < 5; ++f)
#pragma unroll
            for (int j = 0; j < NCH; ++j) acc[j] = fmaf(dec[f], s_w[(F + f) * COUT + lane + 32 * j], acc[j]);
#pragma unroll
        for (int j = 0; j < NCH; ++j) best[j] = fmaxf(best[j], fmaxf(fmaf(acc[j], sc[j], sh[j]), 0.f));
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) out[(size_t)row * COUT + lane + 32 * j] = best[j];
}

}  // namespace

extern "C" int b2s_to_bev(const float *feat, const int *coors, const int *num_rows_dev, int cap_rows, int C,
                          int batch, int D, int H, int W, float *out, int layout, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(C >= 1 && batch >= 1 && D >= 1 && H >= 1 && W >= 1, "b2s_to_bev: bad sizes");
    B2S_REQUIRE(layout == B2S_LAYOUT_NCHW || layout == B2S_LAYOUT_NHWC, "b2s_to_bev: bad layout");
    size_t total = (size_t)batch * C * D * H * W;
    B2S_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * total, stream));
    if (cap_rows > 0) {
        k_to_bev<<<bounded_grid((long long)cap_rows * C), kThreads, 0, stream>>>(
            feat, coors, num_rows_dev, cap_rows, C, batch, D, H, W, out, layout);
        B2S_LAUNCH_OK();
    }
    return 0;
}

extern "C" int b2s_to_bev_tc(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                             const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H,
                             int W, b2s_half *out_hi, b2s_half *out_lo, uint8_t *occupancy, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(C >= 1 && batch >= 1 && D >= 1 && H >= 1 && W >= 1, "b2s_to_bev_tc: bad sizes");
    B2S_REQUIRE((feat != nullptr) != (feat_hi != nullptr && feat_lo != nullptr),
                "b2s_to_bev_tc: pass either fp32 rows or hi/lo fp16 rows");
    size_t total = (size_t)batch * (H + 2) * (W + 2) * C * D;
    B2S_CUDA_OK(cudaMemsetAsync(out_hi, 0, sizeof(__half) * total, stream));
    B2S_CUDA_OK(cudaMemsetAsync(out_lo, 0, sizeof(__half) * total, stream));
    if (occupancy) B2S_CUDA_OK(cudaMemsetAsync(occupancy, 0, (size_t)batch * H * W, stream));
    if (cap_rows > 0) {
        k_to_bev_tc<<<bounded_grid((long long)cap_rows * C), kThreads, 0, stream>>>(
            feat, reinterpret_cast<const __half *>(feat_hi), reinterpret_cast<const __half *>(feat_lo), feat_stride, coors,
            num_rows_dev, cap_rows, C, batch, D, H, W, reinterpret_cast<__half *>(out_hi),
            reinterpret_cast<__half *>(out_lo), occupancy);
        B2S_LAUNCH_OK();
    }
    return 0;
}

extern "C" int b2s_pfn(const float *points, int num_feat, const int *point_slots,
                       const int *num_points_per_voxel, const int *coors, const int *num_rows_dev,
                       int cap_rows, int max_points, const float *weight, const float *scale,
                       const float *shift, int cout, float vx, float vy, float x_offset, float y_offset,
                       float *out, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(num_feat >= 3 && num_feat <= 8, "b2s_pfn: num_feat must be 3..8");
    B2S_REQUIRE(cout == 64, "b2s_pfn: only Cout=64 (PillarFeatureNet num_filters=[64]) is built");
    B2S_REQUIRE(scale != nullptr && shift != nullptr, "b2s_pfn: scale/shift required (BN folded)");
    if (cap_rows == 0) return 0;
    size_t smem = sizeof(float) * (size_t)(num_feat + 5) * cout;
    int warps_per_block = kThreads / 32;
    k_pfn<64><<<b2s_cdiv(cap_rows, warps_per_block), kThreads, smem, stream>>>(
        points, num_feat, point_slots, num_points_per_voxel, coors, num_rows_dev, cap_rows, max_points, weight,
        scale, shift, vx, vy, x_offset, y_offset, out);
    B2S_LAUNCH_OK();
    return 0;
}
