// conv_train.cu -- training of the RPN's 3x3 stride-1 convolutions on the tensor pipe (include/b2second.h, "dense RPN
// training"): the automatically scaled split of an fp32 map into halo-padded fp16 hi/lo planes
// (b2s_split_halo_f16_autoscale) and the weight gradient (b2s_conv2d_wgrad_tc).  The forward and the input gradient are
// b2s_conv2d_tc_ex launches on those planes; the weight planes come from b2s_pack_conv2d_weights (sparse_grad.cu).
//
// Weight gradient: dW[co][ci][ky][kx] = sum_px dY[px][co] * X[px + (ky-1, kx-1)][ci], a GEMM per tap with the pixels as
// its reduction.  Both operands are read by TMA straight from the NHWC halo planes: a box of [pixels, 64 channels]
// with SWIZZLE_128B is the MN-major layout of the 16-bit wgmma (one 128-byte row per pixel, 8 pixel rows per 1024-byte
// atom), so nothing is transposed while staging.  Output strips are 8 pixels wide and 8 rows high (K = 64 pixels).
//
// One CTA owns (2048-pixel slab, dx, 64 input channels, up to 128 output channels).  Per strip a stage holds the
// 10-row x 8-pixel window of X at column offset dx and the strip's dY; the three vertical taps ky are the same window
// ky atoms further on.  So a stage serves three taps, and the two consumer warpgroups (64 output channels each) share
// the X window.  Per tap the chain is 4 k16 steps of dY_hi*X_hi + dY_hi*X_lo + dY_lo*X_hi (12 m64n64k16 MMAs), drained
// into that tap's fp32 running sum with round-to-nearest adds.  The slab partials go to the workspace and a second
// launch adds them in slab order: no float atomics, the result depends on the values and the shape only.
//
// L2 -> SM bytes per pixel: 3 * (Cin/64) * ceil(Cout/128) jobs, each reading X hi/lo (2 x 128 B x 10/8 for the window
// halo) and dY hi/lo (2 x 2 B x min(Cout, 128)); 5.0 KB at 128 -> 128 against 9 KB if each tap re-read both operands.
//
// P = products per k16 step: 3 (3xF16, above) or 1 (the f16 mode, the *_ex entry points with products = 1): one fp16
// plane per operand.  The split writes the hi plane only; the weight gradient's stage holds [X_hi window | dY_hi blocks]
// (half the bytes, 2.5 KB per pixel at 128 -> 128) and each tap's chain is 4 dY_hi*X_hi MMAs.
#include <cuda_fp16.h>

#include "autoscale.cuh"
#include "tc_common.cuh"

namespace {

using namespace b2s_tc;
constexpr int kThreads = 256;
constexpr int WS_R = 8, WS_W = 8;                       // strip: 8 rows x 8 pixels = 64 GEMM K
constexpr int WS_SLAB = 32;                              // strips per slab partial (2048 pixels)
constexpr int WS_STAGES = 3;
constexpr int WS_THREADS = 384;                          // warp 0: TMA producer; warpgroups 1, 2: consumers
constexpr uint32_t ATOM = 1024;                          // 8 pixels x 64 fp16 channels
constexpr uint32_t XWIN_BYTES = (WS_R + 2) * ATOM;       // one plane of the X window
constexpr uint32_t DY_BYTES = WS_R * ATOM;               // one plane of one 64-channel dY block
constexpr uint32_t STAGE_BYTES = 2 * XWIN_BYTES + 4 * DY_BYTES;   // X hi, lo; dY (hi, lo) x 2 blocks
constexpr size_t WS_SMEM = (size_t)WS_STAGES * STAGE_BYTES + 1024;

inline int grid_for(long long items)
{
    long long b = (items + kThreads - 1) / kThreads;
    return (int)(b < 1 ? 1 : (b < 132 * 8 ? b : 132 * 8));
}

inline int num_strips(int B, int H, int W) { return B * ((H + WS_R - 1) / WS_R) * ((W + WS_W - 1) / WS_W); }
inline int num_slabs(int B, int H, int W) { return (num_strips(B, H, W) + WS_SLAB - 1) / WS_SLAB; }

// fp32 map [B, C, H, W] (layout NCHW) or [B, H, W, C] (NHWC) -> x * 2^e as fp16 hi/lo planes [B, H+2, W+2, C] with a zero
// halo.  One thread per (padded pixel, 8 channels); for NCHW consecutive threads take consecutive pixels of one channel
// group, so the reads of each channel row are coalesced.  A non-finite element goes through as itself
// (split_f16_keep_nonfinite) and raises B2S_STATUS_F16_RANGE.  P = 1: the hi plane only.
template <int P>
__global__ void k_split_halo(const float *__restrict__ x, int layout, int B, int C, int H, int W, __half *__restrict__ hi,
                             __half *__restrict__ lo, float *__restrict__ scale_dev, unsigned *__restrict__ status)
{
    const int e = autoscale_exponent(*reinterpret_cast<const volatile unsigned *>(scale_dev + 1));
    const float s = ldexpf(1.f, e);
    if (blockIdx.x == 0 && threadIdx.x == 0) scale_dev[0] = ldexpf(1.f, -e);
    bool nonfinite = false;
    const int G = C / 8, Hp = H + 2, Wp = W + 2;
    const long long n = (long long)B * Hp * Wp * G;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        long long pix;
        int g;
        if (layout == B2S_LAYOUT_NCHW) {                          // i = ((b * G + g) * Hp + hp) * Wp + wp
            const long long q = i / ((long long)Hp * Wp);
            pix = (q / G) * Hp * Wp + (i - q * Hp * Wp);
            g = (int)(q % G);
        } else {                                                  // i = pixel * G + g
            pix = i / G;
            g = (int)(i - pix * G);
        }
        const int wp = (int)(pix % Wp), hp = (int)((pix / Wp) % Hp), b = (int)(pix / ((long long)Hp * Wp));
        uint4 h4 = make_uint4(0, 0, 0, 0), l4 = h4;
        if (hp >= 1 && hp <= H && wp >= 1 && wp <= W) {
            float v[8];
            if (layout == B2S_LAYOUT_NCHW) {
                const size_t plane = (size_t)H * W;
                const float *src = x + ((size_t)b * C + g * 8) * plane + (size_t)(hp - 1) * W + (wp - 1);
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = __ldg(src + j * plane) * s;          // power of two: exact
            } else {
                const float4 *src = reinterpret_cast<const float4 *>(
                    x + (((size_t)b * H + (hp - 1)) * W + (wp - 1)) * C + g * 8);
                const float4 a = __ldg(src), c = __ldg(src + 1);
                v[0] = a.x * s; v[1] = a.y * s; v[2] = a.z * s; v[3] = a.w * s;
                v[4] = c.x * s; v[5] = c.y * s; v[6] = c.z * s; v[7] = c.w * s;
            }
            uint32_t h[4], l[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                nonfinite |= !isfinite(v[2 * j]) || !isfinite(v[2 * j + 1]);
                const uint32_t pa = split_f16_keep_nonfinite(v[2 * j]), pb = split_f16_keep_nonfinite(v[2 * j + 1]);
                h[j] = __byte_perm(pa, pb, 0x5410);
                l[j] = __byte_perm(pa, pb, 0x7632);
            }
            h4 = make_uint4(h[0], h[1], h[2], h[3]);
            l4 = make_uint4(l[0], l[1], l[2], l[3]);
        }
        *reinterpret_cast<uint4 *>(hi + pix * C + g * 8) = h4;
        if constexpr (P == 3) *reinterpret_cast<uint4 *>(lo + pix * C + g * 8) = l4;
    }
    if (nonfinite && status) atomicOr(status, B2S_STATUS_F16_RANGE);
}

// MN-major SWIZZLE_128B descriptor: the 8-row (pixel) groups along K are 1024 B apart.  An operand here is one 64-wide
// MN atom, so the MN-direction offset is never used; both offsets are set to 1024 B.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)(1024 >> 4) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T with both operands MN-major (transpose bits set)
__device__ __forceinline__ void wgmma_mn64(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d));
}

struct WgradParams {
    int B, H, W, Cin, Cout;
    int strips_h, strips_w, strips;
    int ci_blocks, co_pairs;          // job = (dx * ci_blocks + cib) * co_pairs + cop
    float *partial;                   // [slab][tap][Cout][Cin]
};

__device__ __forceinline__ void strip_origin(const WgradParams &p, int id, int &h0, int &w0, int &b)
{
    w0 = (id % p.strips_w) * WS_W;
    h0 = ((id / p.strips_w) % p.strips_h) * WS_R;
    b = id / (p.strips_w * p.strips_h);
}

template <int P>
__global__ void __launch_bounds__(WS_THREADS, 1)
k_conv2d_wgrad_tc(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                  const __grid_constant__ CUtensorMap map_g_hi, const __grid_constant__ CUtensorMap map_g_lo,
                  const WgradParams p)
{
    static_assert(P == 3 || P == 1, "products per k16 step: 3 (3xF16) or 1 (f16)");
    constexpr uint32_t SB = P == 3 ? STAGE_BYTES : XWIN_BYTES + 2 * DY_BYTES;   // P = 1: X_hi, dY_hi x 2 blocks
    constexpr uint32_t XB = (P == 3 ? 2 : 1) * XWIN_BYTES, GB = (P == 3 ? 2 : 1) * DY_BYTES;   // X window, dY block
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t bar_full[WS_STAGES], bar_empty[WS_STAGES];

    const int warp = warp_idx_uniform(), lane = threadIdx.x & 31;
    const int slab = blockIdx.x, job = blockIdx.y;
    const int cop = job % p.co_pairs, cib = (job / p.co_pairs) % p.ci_blocks, dx = job / (p.co_pairs * p.ci_blocks);
    const int s0 = slab * WS_SLAB, s1 = min(s0 + WS_SLAB, p.strips);
    const int co_blocks = min(2, p.Cout / 64 - 2 * cop);     // 64-channel dY blocks of this job (1 or 2)

    if (warp == 1 && lane == 0) {
        for (int i = 0; i < WS_STAGES; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {
            int st = 0;
            uint32_t ph = 0;
            const uint32_t bytes = XB + co_blocks * GB;
            for (int id = s0; id < s1; ++id) {
                int h0, w0, b;
                strip_origin(p, id, h0, w0, b);
                mbar_wait(&bar_empty[st], ph ^ 1);
                uint8_t *dst = smem + (size_t)st * SB;
                mbar_arrive_expect_tx(&bar_full[st], bytes);
                // padded coordinates: output pixel (h, w) of tap (ky, kx) reads X at (h + ky, w + kx), dY at (h+1, w+1);
                // boxes past the padded map are zero-filled, and past-the-edge dY pixels are halo or fill: zero terms
                tma_load_4d(dst, &map_x_hi, &bar_full[st], cib * 64, w0 + dx, h0, b);
                if constexpr (P == 3) tma_load_4d(dst + XWIN_BYTES, &map_x_lo, &bar_full[st], cib * 64, w0 + dx, h0, b);
                for (int q = 0; q < co_blocks; ++q) {
                    const int co = (2 * cop + q) * 64;
                    uint8_t *gd = dst + XB + q * GB;
                    tma_load_4d(gd, &map_g_hi, &bar_full[st], co, w0 + 1, h0 + 1, b);
                    if constexpr (P == 3) tma_load_4d(gd + DY_BYTES, &map_g_lo, &bar_full[st], co, w0 + 1, h0 + 1, b);
                }
                if (++st == WS_STAGES) { st = 0; ph ^= 1; }
            }
        }
    } else if (warp >= 4) {
        const int cg = (warp >> 2) - 1, wl = warp & 3;
        const bool active = cg < co_blocks;
        const uint32_t sm0 = smem_u32(smem);
        float acc[32], sum[3][32];
#pragma unroll
        for (int t = 0; t < 3; ++t)
#pragma unroll
            for (int j = 0; j < 32; ++j) sum[t][j] = 0.f;
        int st = 0;
        uint32_t ph = 0;
        for (int id = s0; id < s1; ++id) {
            mbar_wait(&bar_full[st], ph);
            if (active) {
                const uint32_t sx = sm0 + (uint32_t)st * SB;
                const uint32_t sg = sx + XB + (uint32_t)cg * GB;
#pragma unroll
                for (int ky = 0; ky < 3; ++ky) {
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < WS_R / 2; ++k) {          // k16 step = strip rows 2k, 2k + 1
                        const uint64_t g_hi = make_desc_mn_sw128(sg + 2 * k * ATOM);
                        const uint64_t x_hi = make_desc_mn_sw128(sx + (ky + 2 * k) * ATOM);
                        wgmma_mn64(acc, g_hi, x_hi, k != 0);
                        if constexpr (P == 3) {
                            const uint64_t g_lo = make_desc_mn_sw128(sg + DY_BYTES + 2 * k * ATOM);
                            const uint64_t x_lo = make_desc_mn_sw128(sx + XWIN_BYTES + (ky + 2 * k) * ATOM);
                            wgmma_mn64(acc, g_hi, x_lo, 1);
                            wgmma_mn64(acc, g_lo, x_hi, 1);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait_all();
                    wgmma_fence_operands<32>(acc);
#pragma unroll
                    for (int j = 0; j < 32; ++j) sum[ky][j] = __fadd_rn(sum[ky][j], acc[j]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_empty[st]);
            if (++st == WS_STAGES) { st = 0; ph ^= 1; }
        }
        if (!active) return;
        // accumulator fragment: rows (output channels) 16 wl + lane/4 (+8), columns (input channels) 8j + 2(lane%4)
        const int co_base = (2 * cop + cg) * 64, ci_base = cib * 64;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            float *dst = p.partial + (((size_t)slab * 9 + ky * 3 + dx) * p.Cout) * p.Cin;
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int co = co_base + 16 * wl + (lane >> 2) + 8 * rh;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int ci = ci_base + 8 * j + 2 * (lane & 3);
                    *reinterpret_cast<float2 *>(dst + (size_t)co * p.Cin + ci) =
                        make_float2(sum[ky][4 * j + 2 * rh], sum[ky][4 * j + 2 * rh + 1]);
                }
            }
        }
    }
}

// dw[co][ci][tap] = 2^-(ex + ey) * sum over slabs (ascending) of partial[slab][tap][co][ci]; read in the partial layout
// (coalesced), written with the tap stride of torch's [Cout, Cin, 3, 3]
__global__ void k_conv2d_wgrad_reduce(const float *__restrict__ partial, int slabs, int Cin, int Cout,
                                      const float *__restrict__ x_scale, const float *__restrict__ g_scale,
                                      float *__restrict__ dw)
{
    const int ex = ilogbf(__ldg(x_scale)), eg = ilogbf(__ldg(g_scale));
    const long long elems = 9ll * Cout * Cin;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < elems;
         e += (long long)gridDim.x * blockDim.x) {
        const int ci = (int)(e % Cin), co = (int)((e / Cin) % Cout), tap = (int)(e / ((long long)Cin * Cout));
        float s = 0.f;
        for (int j = 0; j < slabs; ++j) s += __ldg(&partial[(size_t)j * elems + e]);
        dw[((size_t)co * Cin + ci) * 9 + tap] = ldexpf(s, ex + eg);   // one rounding, also into the subnormal range
    }
}

int make_plane_map(CUtensorMap *m, const void *base, int B, int H, int W, int C, int rows)
{
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)(W + 2), (cuuint64_t)(H + 2), (cuuint64_t)B};
    cuuint64_t str[3] = {(cuuint64_t)C * ELEM_BYTES, (cuuint64_t)(W + 2) * C * ELEM_BYTES,
                         (cuuint64_t)(H + 2) * (W + 2) * C * ELEM_BYTES};
    cuuint32_t box[4] = {64, (cuuint32_t)WS_W, (cuuint32_t)rows, 1};
    return make_map(m, base, 4, dims, str, box);
}

}  // namespace

// products = 1: lo must be NULL, only the hi plane is written (the same bits as the hi plane of products = 3)
extern "C" int b2s_split_halo_f16_autoscale_ex(const float *x, int layout, int batch, int C, int H, int W, b2s_half *hi,
                                               b2s_half *lo, float *scale_dev, unsigned *status_dev, int products,
                                               void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && lo == nullptr),
                "b2s_split_halo_f16_autoscale: products must be 3 (hi/lo planes) or 1 (f16, no lo plane)");
    if (products == 1) lo = hi;                       // (the checks below; never written)
    B2S_REQUIRE(layout == B2S_LAYOUT_NCHW || layout == B2S_LAYOUT_NHWC, "b2s_split_halo_f16_autoscale: bad layout");
    B2S_REQUIRE(batch >= 1 && C >= 8 && C % 8 == 0 && H >= 1 && W >= 1,
                "b2s_split_halo_f16_autoscale: bad sizes (C must be a multiple of 8)");
    B2S_REQUIRE((long long)batch * C * H * W < (1ll << 31), "b2s_split_halo_f16_autoscale: map too large");
    B2S_REQUIRE(x && hi && lo && scale_dev, "b2s_split_halo_f16_autoscale: x, hi, lo and scale_dev required");
    B2S_REQUIRE(((uintptr_t)hi & 15) == 0 && ((uintptr_t)lo & 15) == 0 &&
                    (layout == B2S_LAYOUT_NCHW || ((uintptr_t)x & 15) == 0),
                "b2s_split_halo_f16_autoscale: planes (and an NHWC map) must be 16-byte aligned");
    B2S_CUDA_OK(cudaMemsetAsync(scale_dev + 1, 0, sizeof(float), stream));
    const long long n = (long long)batch * C * H * W;
    k_absmax<<<grid_for(n), kThreads, 0, stream>>>(x, nullptr, 1, (int)n, reinterpret_cast<unsigned *>(scale_dev + 1));
    B2S_LAUNCH_OK();
    if (products == 1)
        k_split_halo<1><<<grid_for((long long)batch * (H + 2) * (W + 2) * (C / 8)), kThreads, 0, stream>>>(
            x, layout, batch, C, H, W, reinterpret_cast<__half *>(hi), nullptr, scale_dev, status_dev);
    else
        k_split_halo<3><<<grid_for((long long)batch * (H + 2) * (W + 2) * (C / 8)), kThreads, 0, stream>>>(
            x, layout, batch, C, H, W, reinterpret_cast<__half *>(hi), reinterpret_cast<__half *>(lo), scale_dev,
            status_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_split_halo_f16_autoscale(const float *x, int layout, int batch, int C, int H, int W, b2s_half *hi,
                                            b2s_half *lo, float *scale_dev, unsigned *status_dev, void *stream)
{
    return b2s_split_halo_f16_autoscale_ex(x, layout, batch, C, H, W, hi, lo, scale_dev, status_dev, 3, stream);
}

extern "C" size_t b2s_conv2d_wgrad_tc_workspace_bytes(int batch, int H, int W, int Cin, int Cout)
{
    if (batch <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return 0;
    return sizeof(float) * (size_t)num_slabs(batch, H, W) * 9 * Cin * Cout;
}

// products = 3: the 3xF16 form (b2s_conv2d_wgrad_tc).  products = 1: the f16 mode -- x_lo and dout_lo must be NULL;
// one dY_hi*X_hi product per tap and k16 step, the same workspace.
extern "C" int b2s_conv2d_wgrad_tc_ex(const b2s_half *x_hi, const b2s_half *x_lo, const b2s_half *dout_hi,
                                      const b2s_half *dout_lo, int batch, int H, int W, int Cin, int Cout,
                                      const float *x_scale_dev, const float *dout_scale_dev, float *dweight,
                                      void *workspace, size_t workspace_bytes, int products, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && x_lo == nullptr && dout_lo == nullptr),
                "b2s_conv2d_wgrad_tc: products must be 3 (3xF16) or 1 (f16, no lo planes)");
    if (products == 1) { x_lo = x_hi; dout_lo = dout_hi; }   // (the checks below; never read)
    B2S_REQUIRE(Cin >= 64 && Cin % 64 == 0 && (Cout == 64 || Cout == 128 || Cout == 256),
                "b2s_conv2d_wgrad_tc: Cin must be a multiple of 64 and Cout 64, 128 or 256");
    B2S_REQUIRE(batch >= 1 && H >= 1 && W >= 1, "b2s_conv2d_wgrad_tc: bad sizes");
    B2S_REQUIRE((long long)batch * (H + 2) * (W + 2) * (Cin > Cout ? Cin : Cout) < (1ll << 31),
                "b2s_conv2d_wgrad_tc: map too large");
    B2S_REQUIRE(x_hi && x_lo && dout_hi && dout_lo && x_scale_dev && dout_scale_dev && dweight,
                "b2s_conv2d_wgrad_tc: planes, both scales and dweight required");
    B2S_REQUIRE(((uintptr_t)x_hi & 15) == 0 && ((uintptr_t)x_lo & 15) == 0 && ((uintptr_t)dout_hi & 15) == 0 &&
                    ((uintptr_t)dout_lo & 15) == 0,
                "b2s_conv2d_wgrad_tc: planes must be 16-byte aligned");
    B2S_REQUIRE(workspace_bytes >= b2s_conv2d_wgrad_tc_workspace_bytes(batch, H, W, Cin, Cout),
                "b2s_conv2d_wgrad_tc: workspace too small (b2s_conv2d_wgrad_tc_workspace_bytes)");
    CUtensorMap mx_hi, mx_lo, mg_hi, mg_lo;
    if (make_plane_map(&mx_hi, x_hi, batch, H, W, Cin, WS_R + 2) || make_plane_map(&mg_hi, dout_hi, batch, H, W, Cout, WS_R))
        return -1;
    if (products == 3 && (make_plane_map(&mx_lo, x_lo, batch, H, W, Cin, WS_R + 2) ||
                          make_plane_map(&mg_lo, dout_lo, batch, H, W, Cout, WS_R)))
        return -1;
    WgradParams p;
    p.B = batch; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
    p.strips_h = (H + WS_R - 1) / WS_R;
    p.strips_w = (W + WS_W - 1) / WS_W;
    p.strips = batch * p.strips_h * p.strips_w;
    p.ci_blocks = Cin / 64;
    p.co_pairs = (Cout + 127) / 128;
    p.partial = reinterpret_cast<float *>(workspace);
    const int slabs = num_slabs(batch, H, W);
    if (products == 1) {
        constexpr size_t smem1 = (size_t)WS_STAGES * (XWIN_BYTES + 2 * DY_BYTES) + 1024;
        B2S_SMEM_OPT_IN(k_conv2d_wgrad_tc<1>, smem1);
        k_conv2d_wgrad_tc<1><<<dim3(slabs, 3 * p.ci_blocks * p.co_pairs), WS_THREADS, smem1, stream>>>(mx_hi, mx_hi,
                                                                                                      mg_hi, mg_hi, p);
    } else {
        B2S_SMEM_OPT_IN(k_conv2d_wgrad_tc<3>, WS_SMEM);
        k_conv2d_wgrad_tc<3><<<dim3(slabs, 3 * p.ci_blocks * p.co_pairs), WS_THREADS, WS_SMEM, stream>>>(mx_hi, mx_lo,
                                                                                                        mg_hi, mg_lo, p);
    }
    B2S_LAUNCH_OK();
    k_conv2d_wgrad_reduce<<<grid_for(9ll * Cin * Cout), kThreads, 0, stream>>>(p.partial, slabs, Cin, Cout, x_scale_dev,
                                                                               dout_scale_dev, dweight);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_conv2d_wgrad_tc(const b2s_half *x_hi, const b2s_half *x_lo, const b2s_half *dout_hi,
                                   const b2s_half *dout_lo, int batch, int H, int W, int Cin, int Cout,
                                   const float *x_scale_dev, const float *dout_scale_dev, float *dweight,
                                   void *workspace, size_t workspace_bytes, void *stream)
{
    return b2s_conv2d_wgrad_tc_ex(x_hi, x_lo, dout_hi, dout_lo, batch, H, W, Cin, Cout, x_scale_dev, dout_scale_dev,
                                  dweight, workspace, workspace_bytes, 3, stream);
}
