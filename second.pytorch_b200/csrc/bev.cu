// bev.cu -- sparse rows -> dense BEV map (b2s_to_bev), the PointPillars feature net (b2s_pfn / b2s_pfn_ex) and the
// crop of a halo-padded map into a zero-halo map (b2s_crop_nhwc).  See include/b2second.h.  Pure HBM-bound data movement: zero-fill the dense map once, then one
// scattered write per (row, channel).  b2s_to_bev_tc_ex keeps the map between calls and zeroes only the pixels the
// previous call wrote (7 % of the map for a KITTI cloud), which its occupancy map still flags.
#include <cuda_fp16.h>

#include "pfn_deco.cuh"
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

// tensor-core RPN input: NHWC + one-pixel zero halo, fp16 hi/lo planes (3xF16 split; P = 1: the hi plane only, the
// f16 mode).  The rows come either as fp32 (PointPillars: the PFN output) or already split (the last sparse layer's
// hi/lo planes, row stride feat_stride halves).
template <int P>
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
        if (occ && c == 0) occ[((size_t)q.x * H + q.z) * W + q.w] = 1;      // the pixel holds data (b2s_rpn_block_plan)
        if (feat) {
            const uint32_t pk = b2s_tc::split_f16(__ldg(&feat[gid]));
            out_hi[idx] = __ushort_as_half((unsigned short)(pk & 0xFFFFu));
            if constexpr (P == 3) out_lo[idx] = __ushort_as_half((unsigned short)(pk >> 16));
        } else {
            out_hi[idx] = feat_hi[(size_t)row * feat_stride + c];
            if constexpr (P == 3) out_lo[idx] = feat_lo[(size_t)row * feat_stride + c];
        }
    }
}

// the pixels the previous step flagged in `occ` back to zero in both planes (CV 16-byte vectors per pixel), and their
// flags cleared: each warp reads the flags of 32 pixels and zeroes the flagged ones one pixel at a time (P = 1: the hi
// plane only)
template <int P>
__global__ void k_bev_clear(uint8_t *__restrict__ occ, int batch, int H, int W, int CV, uint4 *__restrict__ out_hi,
                            uint4 *__restrict__ out_lo)
{
    const long long n = (long long)batch * H * W;
    const int lane = threadIdx.x & 31;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long base = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32; base < n; base += nwarps * 32) {
        const long long i = base + lane;
        const bool flagged = i < n && occ[i];
        if (flagged) occ[i] = 0;
        for (unsigned m = __ballot_sync(0xffffffffu, flagged); m; m &= m - 1) {
            const long long px = base + __ffs(m) - 1;
            const long long row = px / W;                                    // b * H + y
            const size_t o = ((size_t)(row + row / H * 2 + 1) * (W + 2) + (px % W) + 1) * CV;
            for (int v = lane; v < CV; v += 32) {
                out_hi[o + v] = make_uint4(0u, 0u, 0u, 0u);
                if constexpr (P == 3) out_lo[o + v] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
    }
}

// PointPillars PFN (single layer): one warp per pillar; lane l owns output channels l, l+32, ...
// decorate each point with (xyz - mean xyz) and (xy - pillar centre), Linear(F+5 -> COUT), BN, ReLU,
// max over the T slots (padded slots contribute relu(shift), exactly like the masked zero rows upstream).
// DECO = B2S_PFN_RADIUS (PillarFeatureNetRadius): the point's own features enter as [|xy|, z, r, ...] instead of
// [x, y, z, r, ...], so the Linear has F+4 inputs.
template <int COUT, int DECO>
__global__ void __launch_bounds__(kThreads)
k_pfn(const float *__restrict__ points, int F, const int *__restrict__ slots, const int *__restrict__ num,
      const int *__restrict__ coors, const int *__restrict__ n_dev, int cap_rows, int T,
      const float *__restrict__ weight, const float *__restrict__ scale, const float *__restrict__ shift,
      float vx, float vy, float xoff, float yoff, float *__restrict__ out)
{
    constexpr int NCH = COUT / 32;
    const int NRAW = DECO == B2S_PFN_RADIUS ? F - 1 : F;    // Linear inputs taken from the point itself
    const int FIN = NRAW + 5;
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
    const auto point = [&](int t) { return points + (size_t)__ldg(&sl[t]) * F; };
    const B2sPfnPillar g = b2s_pfn_pillar(point, np, __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4)),
                                          vx, vy, xoff, yoff);
    float sc[NCH], sh[NCH], best[NCH];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
        sc[j] = __ldg(&scale[lane + 32 * j]);
        sh[j] = __ldg(&shift[lane + 32 * j]);
        // padded slots are all-zero rows upstream: linear -> 0, BN -> shift, ReLU
        best[j] = (np < T) ? fmaxf(sh[j], 0.f) : -INFINITY;
    }
    for (int t = 0; t < np; ++t) {
        float raw[8], dec[5];
        b2s_pfn_decorate<DECO>(point(t), F, g, raw, dec);
        float acc[NCH];
#pragma unroll
        for (int j = 0; j < NCH; ++j) acc[j] = 0.f;
        for (int f = 0; f < NRAW; ++f)
#pragma unroll
            for (int j = 0; j < NCH; ++j) acc[j] = fmaf(raw[f], s_w[f * COUT + lane + 32 * j], acc[j]);
#pragma unroll
        for (int f = 0; f < 5; ++f)
#pragma unroll
            for (int j = 0; j < NCH; ++j) acc[j] = fmaf(dec[f], s_w[(NRAW + f) * COUT + lane + 32 * j], acc[j]);
#pragma unroll
        for (int j = 0; j < NCH; ++j) best[j] = fmaxf(best[j], fmaxf(fmaf(acc[j], sc[j], sh[j]), 0.f));
    }
#pragma unroll
    for (int j = 0; j < NCH; ++j) out[(size_t)row * COUT + lane + 32 * j] = best[j];
}

// interior window [c, H-c) x [c, W-c) of a halo-padded map [B, H+2, W+2, C] -> [B, Ho+2, Wo+2, C] whose halo is
// written as zero; 16-byte vectors (C % 8 == 0); P = 1: the hi plane only
template <int P>
__global__ void k_crop_nhwc(const uint4 *__restrict__ src_hi, const uint4 *__restrict__ src_lo, int batch, int H, int W,
                            int CV, int c, uint4 *__restrict__ dst_hi, uint4 *__restrict__ dst_lo)
{
    const int Ho = H - 2 * c, Wo = W - 2 * c;
    const long long total = (long long)batch * (Ho + 2) * (Wo + 2) * CV;
    for (long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x; gid < total;
         gid += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(gid % CV);
        long long px = gid / CV;
        const int x = (int)(px % (Wo + 2));
        px /= (Wo + 2);
        const int y = (int)(px % (Ho + 2));
        const int b = (int)(px / (Ho + 2));
        uint4 hi = make_uint4(0u, 0u, 0u, 0u), lo = hi;
        if (y >= 1 && y <= Ho && x >= 1 && x <= Wo) {
            // dst interior pixel (y-1, x-1) = src pixel (y-1+c, x-1+c) = padded src (y+c, x+c)
            const size_t s = (((size_t)b * (H + 2) + (y + c)) * (W + 2) + (x + c)) * CV + v;
            hi = __ldg(&src_hi[s]);
            if constexpr (P == 3) lo = __ldg(&src_lo[s]);
        }
        dst_hi[gid] = hi;
        if constexpr (P == 3) dst_lo[gid] = lo;
    }
}

template <int DECO>
int pfn_launch(const float *points, int num_feat, const int *point_slots, const int *num_points_per_voxel,
               const int *coors, const int *num_rows_dev, int cap_rows, int max_points, const float *weight,
               const float *scale, const float *shift, int cout, float vx, float vy, float x_offset, float y_offset,
               float *out, cudaStream_t stream)
{
    const int fin = num_feat + (DECO == B2S_PFN_RADIUS ? 4 : 5);
    size_t smem = sizeof(float) * (size_t)fin * cout;
    int warps_per_block = kThreads / 32;
    k_pfn<64, DECO><<<b2s_cdiv(cap_rows, warps_per_block), kThreads, smem, stream>>>(
        points, num_feat, point_slots, num_points_per_voxel, coors, num_rows_dev, cap_rows, max_points, weight,
        scale, shift, vx, vy, x_offset, y_offset, out);
    B2S_LAUNCH_OK();
    return 0;
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
        k_to_bev_tc<3><<<bounded_grid((long long)cap_rows * C), kThreads, 0, stream>>>(
            feat, reinterpret_cast<const __half *>(feat_hi), reinterpret_cast<const __half *>(feat_lo), feat_stride, coors,
            num_rows_dev, cap_rows, C, batch, D, H, W, reinterpret_cast<__half *>(out_hi),
            reinterpret_cast<__half *>(out_lo), occupancy);
        B2S_LAUNCH_OK();
    }
    return 0;
}

// products = 3: hi/lo planes; products = 1 (the f16 mode): feat_lo and out_lo must be NULL, one fp16 plane
extern "C" int b2s_to_bev_tc_ex2(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                                 const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H,
                                 int W, b2s_half *out_hi, b2s_half *out_lo, uint8_t *occupancy, int products,
                                 void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && feat_lo == nullptr && out_lo == nullptr),
                "b2s_to_bev_tc_ex: products must be 3 (hi/lo planes) or 1 (f16, no lo planes)");
    B2S_REQUIRE(C >= 1 && batch >= 1 && D >= 1 && H >= 1 && W >= 1, "b2s_to_bev_tc_ex: bad sizes");
    B2S_REQUIRE((feat != nullptr) != (feat_hi != nullptr && (feat_lo != nullptr || products == 1)),
                "b2s_to_bev_tc_ex: pass either fp32 rows or hi/lo fp16 rows");
    B2S_REQUIRE(occupancy != nullptr && (C * D) % 8 == 0 && ((uintptr_t)out_hi & 15) == 0 && ((uintptr_t)out_lo & 15) == 0,
                "b2s_to_bev_tc_ex: needs the occupancy map, C*D a multiple of 8 and 16-byte aligned planes");
    const int grid_clear = bounded_grid((long long)batch * H * W), grid_rows = bounded_grid((long long)cap_rows * C);
    const __half *fh = reinterpret_cast<const __half *>(feat_hi), *fl = reinterpret_cast<const __half *>(feat_lo);
    __half *oh = reinterpret_cast<__half *>(out_hi), *ol = reinterpret_cast<__half *>(out_lo);
    if (products == 1)
        k_bev_clear<1><<<grid_clear, kThreads, 0, stream>>>(occupancy, batch, H, W, C * D / 8,
                                                            reinterpret_cast<uint4 *>(oh), nullptr);
    else
        k_bev_clear<3><<<grid_clear, kThreads, 0, stream>>>(occupancy, batch, H, W, C * D / 8,
                                                            reinterpret_cast<uint4 *>(oh), reinterpret_cast<uint4 *>(ol));
    B2S_LAUNCH_OK();
    if (cap_rows > 0) {
        if (products == 1)
            k_to_bev_tc<1><<<grid_rows, kThreads, 0, stream>>>(feat, fh, nullptr, feat_stride, coors, num_rows_dev,
                                                               cap_rows, C, batch, D, H, W, oh, nullptr, occupancy);
        else
            k_to_bev_tc<3><<<grid_rows, kThreads, 0, stream>>>(feat, fh, fl, feat_stride, coors, num_rows_dev, cap_rows,
                                                               C, batch, D, H, W, oh, ol, occupancy);
        B2S_LAUNCH_OK();
    }
    return 0;
}

extern "C" int b2s_to_bev_tc_ex(const float *feat, const b2s_half *feat_hi, const b2s_half *feat_lo, int feat_stride,
                                const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch, int D, int H,
                                int W, b2s_half *out_hi, b2s_half *out_lo, uint8_t *occupancy, void *stream)
{
    return b2s_to_bev_tc_ex2(feat, feat_hi, feat_lo, feat_stride, coors, num_rows_dev, cap_rows, C, batch, D, H, W,
                             out_hi, out_lo, occupancy, 3, stream);
}

extern "C" int b2s_pfn(const float *points, int num_feat, const int *point_slots,
                       const int *num_points_per_voxel, const int *coors, const int *num_rows_dev,
                       int cap_rows, int max_points, const float *weight, const float *scale,
                       const float *shift, int cout, float vx, float vy, float x_offset, float y_offset,
                       float *out, void *stream_)
{
    return b2s_pfn_ex(points, num_feat, point_slots, num_points_per_voxel, coors, num_rows_dev, cap_rows, max_points,
                      weight, scale, shift, cout, vx, vy, x_offset, y_offset, B2S_PFN_PLAIN, out, stream_);
}

extern "C" int b2s_pfn_ex(const float *points, int num_feat, const int *point_slots,
                          const int *num_points_per_voxel, const int *coors, const int *num_rows_dev,
                          int cap_rows, int max_points, const float *weight, const float *scale,
                          const float *shift, int cout, float vx, float vy, float x_offset, float y_offset,
                          int decoration, float *out, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(num_feat >= 3 && num_feat <= 8, "b2s_pfn: num_feat must be 3..8");
    B2S_REQUIRE(cout == 64, "b2s_pfn: only Cout=64 (PillarFeatureNet num_filters=[64]) is built");
    B2S_REQUIRE(scale != nullptr && shift != nullptr, "b2s_pfn: scale/shift required (BN folded)");
    B2S_REQUIRE(decoration == B2S_PFN_PLAIN || decoration == B2S_PFN_RADIUS,
                "b2s_pfn_ex: decoration must be B2S_PFN_PLAIN (0) or B2S_PFN_RADIUS (1)");
    if (cap_rows == 0) return 0;
    if (decoration == B2S_PFN_RADIUS)
        return pfn_launch<B2S_PFN_RADIUS>(points, num_feat, point_slots, num_points_per_voxel, coors, num_rows_dev,
                                          cap_rows, max_points, weight, scale, shift, cout, vx, vy, x_offset, y_offset,
                                          out, stream);
    return pfn_launch<B2S_PFN_PLAIN>(points, num_feat, point_slots, num_points_per_voxel, coors, num_rows_dev, cap_rows,
                                     max_points, weight, scale, shift, cout, vx, vy, x_offset, y_offset, out, stream);
}

// products = 3: hi/lo planes; products = 1 (the f16 mode): src_lo and dst_lo must be NULL, one fp16 plane
extern "C" int b2s_crop_nhwc_ex(const b2s_half *src_hi, const b2s_half *src_lo, int batch, int H, int W, int C, int crop,
                                b2s_half *dst_hi, b2s_half *dst_lo, int products, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && src_lo == nullptr && dst_lo == nullptr),
                "b2s_crop_nhwc: products must be 3 (hi/lo planes) or 1 (f16, no lo planes)");
    B2S_REQUIRE(batch >= 1 && H >= 1 && W >= 1 && crop >= 0 && H - 2 * crop >= 1 && W - 2 * crop >= 1,
                "b2s_crop_nhwc: bad sizes (the window [crop, H-crop) x [crop, W-crop) must be non-empty)");
    B2S_REQUIRE(C % 8 == 0 && ((uintptr_t)src_hi & 15) == 0 && ((uintptr_t)src_lo & 15) == 0 &&
                    ((uintptr_t)dst_hi & 15) == 0 && ((uintptr_t)dst_lo & 15) == 0,
                "b2s_crop_nhwc: C must be a multiple of 8 and the planes 16-byte aligned");
    const long long total = (long long)batch * (H - 2 * crop + 2) * (W - 2 * crop + 2) * (C / 8);
    if (products == 1)
        k_crop_nhwc<1><<<bounded_grid(total), kThreads, 0, stream>>>(
            reinterpret_cast<const uint4 *>(src_hi), nullptr, batch, H, W, C / 8, crop, reinterpret_cast<uint4 *>(dst_hi),
            nullptr);
    else
        k_crop_nhwc<3><<<bounded_grid(total), kThreads, 0, stream>>>(
            reinterpret_cast<const uint4 *>(src_hi), reinterpret_cast<const uint4 *>(src_lo), batch, H, W, C / 8, crop,
            reinterpret_cast<uint4 *>(dst_hi), reinterpret_cast<uint4 *>(dst_lo));
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_crop_nhwc(const b2s_half *src_hi, const b2s_half *src_lo, int batch, int H, int W, int C, int crop,
                             b2s_half *dst_hi, b2s_half *dst_lo, void *stream)
{
    return b2s_crop_nhwc_ex(src_hi, src_lo, batch, H, W, C, crop, dst_hi, dst_lo, 3, stream);
}
