// conv_tc.cu -- dense RPN convolution as a wgmma implicit GEMM with fp32-grade accuracy (b2s_conv2d_tc).
//
// second.pytorch's RPNV2 (second/pytorch/models/rpn.py:467-497, forward :314-331,393-420) is a stack of
// Conv2d(3x3, pad 1)+BatchNorm2d+ReLU blocks, 1x1 (de)conv blocks and 1x1 heads: 63.6 GFLOP/frame at car.fhd,
// the FLOP majority of the frame.  cuDNN runs it in fp32 SIMT (the parity bar is fp32, TF32 is off).  Here it is
//
//     D[M = 128 pixels, N = Cout] += A[M, K = 64 channels of one tap] * B[N, K]^T        (wgmma, f16 -> f32)
//
// with the **3xF16 split** (tc_common.cuh) that keeps fp32-grade accuracy on the tensor pipe: every operand is stored
// as hi = fp16(x) and lo = fp16(x - hi), and each K step issues
//     A_lo*B_hi + A_hi*B_lo + A_hi*B_hi            (the dropped A_lo*B_lo term is ~2^-22 relative)
// accumulating in fp32 registers.
//
// Layout: activations NHWC fp16 with a one-pixel zero halo, [B, H+2, W+2, C] (hi and lo planes), so every
// filter tap is a plain shifted box and TMA (cp.async.bulk.tensor.4d, SWIZZLE_128B) fetches the
// [8 rows x 16 cols x 64 channels] A tile of a tap directly into the K-major wgmma layout; image borders come
// from the halo, partial tiles from TMA's out-of-bounds zero fill.  Weights are pre-arranged [tap][Cout][Cin].
//
// CTA = 3 warpgroups, persistent over output tiles (static round robin):
//   warp 0       TMA producer: per K block (tap, 64-channel chunk) 4 bulk-tensor loads into a STAGES-deep smem ring
//   warpgroups 1, 2  consumers: warpgroup g issues the wgmmas of tile rows 64g .. 64g+63 and owns their accumulators;
//                then BN scale/shift -> ReLU -> hi/lo split -> NHWC stores
// The ring's full/empty mbarriers let the loads of the next K blocks (and of the next tile) run under the MMAs.
//
// Every mbarrier wait is bounded: on a (never expected) protocol error the kernel traps instead of hanging the GPU.
//
// P = products per K step: 3 is the 3xF16 split above; 1 is the f16 mode (b2s_conv2d_tc_ex3 with products = 1): one
// fp16 plane per operand, so a stage holds the A and B hi tiles only, each K step is one wgmma A_hi*B_hi, and the
// epilogue writes one rounded fp16 plane, or with F32_OUT the fp32 result (P = 3 reads that from out_lo == NULL).
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

using namespace b2s_tc;
constexpr int TILE_H = 8, TILE_W = 16;   // BLOCK_M = 128 output pixels = 8 rows x 16 cols
constexpr int kThreads = 384;

struct ConvParams {
    int B, H, W;             // the GEMM pixel grid: conv output pixels (for a k=s deconv sub-grid: the input pixels)
    int Cin, Cout, taps, relu;
    int kw;                  // filter width (tap = dy*kw + dx)
    int stride;              // input pixel step per GEMM pixel (TMA element stride)
    int in_off;              // 1 - padding: halo-padded input coordinate of GEMM pixel 0, tap 0
    int tiles_h, tiles_w, num_tiles;
    int Hout, Wout;          // output map size; GEMM pixel (h,w) is written to (h*out_mul+off_h, w*out_mul+off_w)
    int out_mul, off_h, off_w;
    int out_padded;          // 1: out is [B,Hout+2,Wout+2,*] (interior written), 0: [B,Hout,Wout,*]
    int out_stride;          // channels per output pixel row (>= Cout; lets heads write a packed record)
    const float *scale, *shift;
    void *out_hi;            // fp16 hi plane, or (out_lo == NULL) the full fp32 result
    __half *out_lo;
    int *status;
};

// The statements of the 3xF16 instances are kept as they were (their SASS is unchanged by the f16 instances): what
// only the 3xF16 form does goes through these helpers, which compile to nothing for the f16 form.
template <bool ON>
__device__ __forceinline__ void tma_load_4d_if(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2,
                                               int c3)
{
    if constexpr (ON) tma_load_4d(dst, map, bar, c0, c1, c2, c3);
}
template <bool ON>
__device__ __forceinline__ void tma_load_3d_if(void *dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2)
{
    if constexpr (ON) tma_load_3d(dst, map, bar, c0, c1, c2);
}
template <bool ON>
__device__ __forceinline__ void store_u32_if(__half *dst, uint32_t v)
{
    if constexpr (ON) *reinterpret_cast<uint32_t *>(dst) = v;
}
// the epilogue writes fp16 planes: 3xF16 when out_lo is given, f16 unless the instance writes fp32
template <int P, bool F32_OUT>
__device__ __forceinline__ bool f16_planes_out(const __half *out_lo)
{
    if constexpr (P == 3) return out_lo != nullptr;
    else return !F32_OUT;
}

template <int N, int STAGES, int P, bool F32_OUT>
__global__ void __launch_bounds__(kThreads, 1)
k_conv_tc(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
          const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
          const ConvParams p)
{
    constexpr uint32_t B_TILE_BYTES = N * BLOCK_K * ELEM_BYTES;
    static_assert(P == 3 || P == 1, "products per K step: 3 (3xF16) or 1 (f16)");
    constexpr uint32_t STAGE_BYTES = P == 3 ? 2 * A_TILE_BYTES + 2 * B_TILE_BYTES : A_TILE_BYTES + B_TILE_BYTES;
    constexpr int R = N / 2;                 // accumulator registers per thread (64 rows x N per warpgroup)
    // The tensor core's fp32 accumulate is not round-to-nearest: one long accumulation chain (432 MMAs for a 3x3x128
    // tap stack) carries a systematic ~2e-5 relative error.  So the reduction is cut into short chains of CHAIN K
    // blocks (tap x 64-channel chunk; 4 = 48 MMAs), and each chain's partial sum is added to the running fp32 sum with
    // round-to-nearest.
    constexpr int CHAIN = 4;
    static_assert(N % 16 == 0 && N >= 16 && N <= 128, "wgmma N");

    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t bar_full[STAGES], bar_empty[STAGES];
    __shared__ float s_scale[N], s_shift[N];

    const int warp = warp_idx_uniform(), lane = threadIdx.x & 31;
    const int kchunks = p.Cin / BLOCK_K;
    const int num_kb = p.taps * kchunks;

    if (threadIdx.x < N) {
        int c = threadIdx.x;
        s_scale[c] = (p.scale && c < p.Cout) ? p.scale[c] : 1.f;
        s_shift[c] = (p.shift && c < p.Cout) ? p.shift[c] : 0.f;
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&bar_full[i], 1); mbar_init(&bar_empty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
                int tw = tile % p.tiles_w;
                int th = (tile / p.tiles_w) % p.tiles_h;
                int b = tile / (p.tiles_w * p.tiles_h);
                // halo-padded input coordinate of the tile's first GEMM pixel; the tensor map's element stride
                // (= p.stride) makes the 16 x 8 box step over the input pixels of a strided conv
                const int h0 = th * TILE_H * p.stride + p.in_off, w0 = tw * TILE_W * p.stride + p.in_off;
                for (int kb = 0; kb < num_kb; ++kb) {
                    int tap = kb / kchunks, chunk = kb - tap * kchunks;
                    const int dy = tap / p.kw, dx = tap - dy * p.kw;
                    mbar_wait(&bar_empty[stage], phase ^ 1);
                    uint8_t *st = smem + (size_t)stage * STAGE_BYTES;
                    mbar_arrive_expect_tx(&bar_full[stage], STAGE_BYTES);
                    // 3xF16: [A_hi | A_lo | B_hi | B_lo]; f16: [A_hi | B_hi]
                    tma_load_4d(st, &map_a_hi, &bar_full[stage], chunk * BLOCK_K, w0 + dx, h0 + dy, b);
                    tma_load_4d_if<P == 3>(st + A_TILE_BYTES, &map_a_lo, &bar_full[stage], chunk * BLOCK_K, w0 + dx,
                                           h0 + dy, b);
                    tma_load_3d(st + (P == 3 ? 2 : 1) * A_TILE_BYTES, &map_b_hi, &bar_full[stage], chunk * BLOCK_K, 0, tap);
                    tma_load_3d_if<P == 3>(st + 2 * A_TILE_BYTES + B_TILE_BYTES, &map_b_lo, &bar_full[stage],
                                           chunk * BLOCK_K, 0, tap);
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else if (warp >= 4) {
        // ===================== consumers: MMA + epilogue =====================
        const int cg = (warp >> 2) - 1;          // warpgroup 0 / 1: tile rows 64 cg .. 64 cg + 63
        const int wl = warp & 3;
        const uint32_t smem0 = smem_u32(smem);
        const uint32_t a_off = (uint32_t)cg * 64u * 128u;
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
            int tw = tile % p.tiles_w;
            int th = (tile / p.tiles_w) % p.tiles_h;
            int b = tile / (p.tiles_w * p.tiles_h);
            float sum[R], acc[R];
#pragma unroll
            for (int j = 0; j < R; ++j) sum[j] = 0.f;
            // accumulation chains of CHAIN K blocks, whatever the tap / channel split
            for (int kb0 = 0; kb0 < num_kb; kb0 += CHAIN) {
                const int kb_chain = min(num_kb, kb0 + CHAIN) - kb0;
                for (int chunk = 0; chunk < kb_chain; ++chunk) {
                    mbar_wait(&bar_full[stage], phase);          // TMA bytes have landed
                    const uint32_t sa = smem0 + (uint32_t)stage * STAGE_BYTES;
                    if constexpr (P == 3) {
                        const uint64_t a_hi = make_desc_sw128(sa + a_off), a_lo = make_desc_sw128(sa + A_TILE_BYTES + a_off);
                        const uint64_t b_hi = make_desc_sw128(sa + 2 * A_TILE_BYTES);
                        const uint64_t b_lo = make_desc_sw128(sa + 2 * A_TILE_BYTES + B_TILE_BYTES);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
                            const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);   // +32 B per K step
                            wgmma_ss<N>(acc, a_lo + koff, b_hi + koff, (chunk | k) != 0);
                            wgmma_ss<N>(acc, a_hi + koff, b_lo + koff, 1);
                            wgmma_ss<N>(acc, a_hi + koff, b_hi + koff, 1);
                        }
                    } else {
                        const uint64_t a_hi = make_desc_sw128(sa + a_off), b_hi = make_desc_sw128(sa + A_TILE_BYTES);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
                            const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                            wgmma_ss<N>(acc, a_hi + koff, b_hi + koff, (chunk | k) != 0);
                        }
                    }
                    wgmma_commit();
                    wgmma_wait_all();
                    wgmma_fence_operands<R>(acc);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bar_empty[stage]);    // this warp's share of the stage has been read
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
                // drain the chain's partial sum into the fp32 running sum (round-to-nearest adds)
#pragma unroll
                for (int j = 0; j < R; ++j) sum[j] = __fadd_rn(sum[j], acc[j]);
            }
            // epilogue: this thread holds rows m0 = 64 cg + 16 wl + lane/4 and m0 + 8, and per 8-column block j the
            // channel pair 8j + 2(lane % 4); a quad of lanes writes 16 (fp16 plane) or 32 (fp32) contiguous bytes
            bool range_bad = false;
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int mm = cg * 64 + wl * 16 + (lane >> 2) + rh * 8;
                const int hh = th * TILE_H + mm / TILE_W, ww = tw * TILE_W + mm % TILE_W;
                if (hh >= p.H || ww >= p.W) continue;
                const int oh = hh * p.out_mul + p.off_h, ow = ww * p.out_mul + p.off_w;   // position in the output map
                const size_t gpix = p.out_padded ? ((size_t)b * (p.Hout + 2) + (oh + 1)) * (p.Wout + 2) + (ow + 1)
                                                 : ((size_t)b * p.Hout + oh) * p.Wout + ow;
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    if (c >= p.Cout) continue;                   // Cout is a multiple of 4: c + 1 < Cout too
                    float x0 = fmaf(sum[4 * j + 2 * rh], s_scale[c], s_shift[c]);
                    float x1 = fmaf(sum[4 * j + 2 * rh + 1], s_scale[c + 1], s_shift[c + 1]);
                    if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                    if (f16_planes_out<P, F32_OUT>(p.out_lo)) {
                        range_bad |= (fabsf(x0) > 65504.f) | (fabsf(x1) > 65504.f);
                        const uint32_t p0 = split_f16(x0), p1 = split_f16(x1);
                        *reinterpret_cast<uint32_t *>(reinterpret_cast<__half *>(p.out_hi) + gpix * p.out_stride + c) =
                            __byte_perm(p0, p1, 0x5410);
                        store_u32_if<P == 3>(p.out_lo + gpix * p.out_stride + c, __byte_perm(p0, p1, 0x7632));
                    } else {
                        *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out_hi) + gpix * p.out_stride + c) =
                            make_float2(x0, x1);
                    }
                }
            }
            if (__any_sync(0xffffffffu, range_bad) && lane == 0 && p.status) atomicOr(p.status, B2S_STATUS_F16_RANGE);
        }
    }
}

template <int N, int STAGES, int P, bool F32_OUT = false>
int launch(const CUtensorMap &a_hi, const CUtensorMap &a_lo, const CUtensorMap &b_hi, const CUtensorMap &b_lo,
           const ConvParams &p, int num_sms, cudaStream_t stream)
{
    constexpr size_t stage = (P == 3 ? 2 : 1) * (A_TILE_BYTES + (size_t)N * BLOCK_K * ELEM_BYTES);
    size_t smem = stage * STAGES + 1024;
    B2S_SMEM_OPT_IN((k_conv_tc<N, STAGES, P, F32_OUT>), smem);
    int grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
    k_conv_tc<N, STAGES, P, F32_OUT><<<grid, kThreads, smem, stream>>>(a_hi, a_lo, b_hi, b_lo, p);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

// conv_tc2.cu
int b2s_conv3x3_tc2(const __half *in_hi, const __half *in_lo, int B, int H, int W, int Cin, const __half *w_hi,
                    const __half *w_lo, int Cout, const float *scale, const float *shift, int relu, __half *out_hi,
                    __half *out_lo, int out_stride, const int *work_list, const int *work_count, const int *bg_list,
                    const int *bg_count, const __half *bg_hi, const __half *bg_lo, int bg_margin, int list_rows,
                    int products, int *status, int num_sms, cudaStream_t stream);

// General form (include/b2second.h).  Input: halo-padded fp16 hi/lo planes [B, Hin+2, Win+2, Cin].  One GEMM pixel
// (h, w) of the Hg x Wg grid reads input pixels (h*stride + dy - pad, w*stride + dx - pad), dy < kh, dx < kw, and is
// written to output pixel (h*out_mul + off_h, w*out_mul + off_w) of an Hout x Wout map:
//   conv  k x k, stride s, pad p : Hg = Hout = conv output size, out_mul 1
//   ConvTranspose2d k = s        : s*s launches with kh = kw = 1, Hg = Hin, out_mul = s, (off_h, off_w) = (a, c),
//                                  weights W[:, :, a, c]
// work_list / bg_list name output strips 8 wide and list_rows (8, 4 or 2) high (b2s_rpn_block_plan,
// b2s_rpn_strip_plan).  bg_margin >= 0: the field bg_hi/bg_lo equals its value at pixel (bg_margin, bg_margin)
// wherever it is at least bg_margin pixels from every border, and background strips there are stored from that value.
//
// products = 3: 3xF16 (hi/lo planes; out_lo == NULL: fp32 output).  products = 1: the f16 mode -- every lo pointer
// (in_lo, w_lo, out_lo, bg_lo) must be NULL, the output is one fp16 plane in out_hi, or the fp32 result when out_fp32
// is 1 (out_fp32 must be 0 with products = 3, where out_lo says it).
extern "C" int b2s_conv2d_tc_ex3(const b2s_half *in_hi_, const b2s_half *in_lo_, int B, int Hin, int Win, int Cin,
                                 const b2s_half *w_hi_, const b2s_half *w_lo_, int kh, int kw, int stride, int pad,
                                 int Cout, int n_pad, const float *scale, const float *shift, int relu, int Hg, int Wg,
                                 void *out_hi, b2s_half *out_lo_, int Hout, int Wout, int out_padded, int out_stride,
                                 int out_mul, int off_h, int off_w, const int *work_list, const int *work_count_dev,
                                 const int *bg_list, const int *bg_count_dev, const b2s_half *bg_hi,
                                 const b2s_half *bg_lo, int bg_margin, int list_rows, int products, int out_fp32,
                                 unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    const __half *in_hi = reinterpret_cast<const __half *>(in_hi_), *in_lo = reinterpret_cast<const __half *>(in_lo_);
    const __half *w_hi = reinterpret_cast<const __half *>(w_hi_), *w_lo = reinterpret_cast<const __half *>(w_lo_);
    __half *out_lo = reinterpret_cast<__half *>(out_lo_);
    const int taps = kh * kw;
    B2S_REQUIRE(products == 3 || products == 1, "b2s_conv2d_tc: products must be 3 (3xF16) or 1 (f16)");
    B2S_REQUIRE(products == 3 ? out_fp32 == 0
                              : (in_lo == nullptr && w_lo == nullptr && out_lo == nullptr && bg_lo == nullptr &&
                                 (out_fp32 == 0 || out_fp32 == 1)),
                "b2s_conv2d_tc: products = 1 takes no lo planes and out_fp32 0 or 1; products = 3 takes out_fp32 = 0");
    // fp16 plane output: hi/lo (products 3, out_lo given) or one plane (products 1, out_fp32 0)
    const bool f16_out = products == 3 ? out_lo != nullptr : out_fp32 == 0;
    B2S_REQUIRE(kh >= 1 && kw >= 1 && taps <= 16 && stride >= 1 && stride <= 4 && (pad == 0 || pad == 1),
                "b2s_conv2d_tc: kernel up to 4x4 (16 taps), stride 1..4, pad 0 or 1");
    B2S_REQUIRE(Cin % BLOCK_K == 0 && Cin >= BLOCK_K, "b2s_conv2d_tc: Cin must be a multiple of 64");
    B2S_REQUIRE(n_pad >= Cout && Cout % 4 == 0 && out_stride >= Cout && out_stride % 4 == 0,
                "b2s_conv2d_tc: Cout/out_stride must be multiples of 4, n_pad >= Cout");
    B2S_REQUIRE(!f16_out || (Cout % 8 == 0 && out_stride % 8 == 0 && ((uintptr_t)out_hi & 15) == 0 &&
                             ((uintptr_t)out_lo & 15) == 0),
                "b2s_conv2d_tc: fp16 plane output needs Cout, out_stride multiples of 8 and 16-byte aligned pointers");
    B2S_REQUIRE(B >= 1 && Hin >= 1 && Win >= 1 && Hg >= 1 && Wg >= 1 && out_mul >= 1, "b2s_conv2d_tc: bad sizes");
    B2S_REQUIRE((Hg - 1) * out_mul + off_h < Hout && (Wg - 1) * out_mul + off_w < Wout && off_h >= 0 && off_w >= 0,
                "b2s_conv2d_tc: output positions outside the Hout x Wout map");
    const int num_sms = num_sms_current();
    // 3x3 stride 1 pad 1, n_pad 128, hi/lo halo-padded output on the same grid: the weights-stationary N=256
    // kernel (conv_tc2.cu).  Every other shape runs k_conv_tc below.
    const bool v2 = kh == 3 && kw == 3 && stride == 1 && pad == 1 && n_pad == 128 && f16_out &&
                    out_padded && out_mul == 1 && off_h == 0 && off_w == 0 && Hg == Hin && Wg == Win && Hout == Hin &&
                    Wout == Win;
    B2S_REQUIRE(work_list == nullptr || (v2 && work_count_dev != nullptr),
                "b2s_conv2d_tc: a strip work list is only taken by the 3x3 stride-1 128-channel kernel");
    B2S_REQUIRE(work_list == nullptr || list_rows == 8 || list_rows == 4 || list_rows == 2,
                "b2s_conv2d_tc: work-list strips are 8, 4 or 2 rows high");
    B2S_REQUIRE(bg_list == nullptr || (work_list != nullptr && bg_count_dev != nullptr && bg_hi != nullptr &&
                                       (bg_lo != nullptr || products == 1)),
                "b2s_conv2d_tc: a background-block list needs the work list, its count and the constant's hi/lo planes");
    if (v2)
        return b2s_conv3x3_tc2(in_hi, in_lo, B, Hin, Win, Cin, w_hi, w_lo, Cout, scale, shift, relu,
                               reinterpret_cast<__half *>(out_hi), out_lo, out_stride, work_list, work_count_dev, bg_list,
                               bg_count_dev, reinterpret_cast<const __half *>(bg_hi), reinterpret_cast<const __half *>(bg_lo),
                               bg_margin, list_rows, products, (int *)status_dev, num_sms, stream);
    CUtensorMap a_hi, a_lo, b_hi, b_lo;
    {
        cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)(Win + 2), (cuuint64_t)(Hin + 2), (cuuint64_t)B};
        cuuint64_t str[3] = {(cuuint64_t)Cin * ELEM_BYTES, (cuuint64_t)(Win + 2) * Cin * ELEM_BYTES,
                             (cuuint64_t)(Hin + 2) * (Win + 2) * Cin * ELEM_BYTES};
        // the box TRAVERSES stride*TILE pixels and keeps every stride-th one: TILE_W x TILE_H pixels land in smem
        cuuint32_t box[4] = {BLOCK_K, (cuuint32_t)(TILE_W * stride), (cuuint32_t)(TILE_H * stride), 1};
        cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
        if (make_map(&a_hi, in_hi, 4, dims, str, box, es) ||
            (products == 3 && make_map(&a_lo, in_lo, 4, dims, str, box, es)))
            return -1;
    }
    {
        // weights [taps][n_pad][Cin] (rows >= Cout are zero)
        cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)n_pad, (cuuint64_t)taps};
        cuuint64_t str[2] = {(cuuint64_t)Cin * ELEM_BYTES, (cuuint64_t)n_pad * Cin * ELEM_BYTES};
        cuuint32_t box[3] = {BLOCK_K, (cuuint32_t)n_pad, 1};
        if (make_map(&b_hi, w_hi, 3, dims, str, box) || (products == 3 && make_map(&b_lo, w_lo, 3, dims, str, box)))
            return -1;
    }
    ConvParams p;
    p.B = B; p.H = Hg; p.W = Wg; p.Cin = Cin; p.Cout = Cout; p.taps = taps; p.relu = relu;
    p.kw = kw; p.stride = stride; p.in_off = 1 - pad;
    p.tiles_h = (Hg + TILE_H - 1) / TILE_H;
    p.tiles_w = (Wg + TILE_W - 1) / TILE_W;
    p.num_tiles = B * p.tiles_h * p.tiles_w;
    p.Hout = Hout; p.Wout = Wout; p.out_mul = out_mul; p.off_h = off_h; p.off_w = off_w;
    p.out_padded = out_padded; p.out_stride = out_stride;
    p.scale = scale; p.shift = shift; p.out_hi = out_hi; p.out_lo = out_lo; p.status = (int *)status_dev;
    if (products == 1 && f16_out) {
        switch (n_pad) {
            case 128: return launch<128, 3, 1>(a_hi, a_hi, b_hi, b_hi, p, num_sms, stream);
            case 64: return launch<64, 4, 1>(a_hi, a_hi, b_hi, b_hi, p, num_sms, stream);
            case 32: return launch<32, 4, 1>(a_hi, a_hi, b_hi, b_hi, p, num_sms, stream);
            default: break;
        }
    } else if (products == 1) {
        switch (n_pad) {
            case 128: return launch<128, 3, 1, true>(a_hi, a_hi, b_hi, b_hi, p, num_sms, stream);
            case 64: return launch<64, 4, 1, true>(a_hi, a_hi, b_hi, b_hi, p, num_sms, stream);
            case 32: return launch<32, 4, 1, true>(a_hi, a_hi, b_hi, b_hi, p, num_sms, stream);
            default: break;
        }
    } else {
        switch (n_pad) {
            case 128: return launch<128, 3, 3>(a_hi, a_lo, b_hi, b_lo, p, num_sms, stream);
            case 64: return launch<64, 4, 3>(a_hi, a_lo, b_hi, b_lo, p, num_sms, stream);
            case 32: return launch<32, 4, 3>(a_hi, a_lo, b_hi, b_lo, p, num_sms, stream);
            default: break;
        }
    }
    b2s_set_error("b2s_conv2d_tc: n_pad=%d not built (32, 64, 128)", n_pad);
    return -2;
}

// the 3xF16 form
extern "C" int b2s_conv2d_tc_ex2(const b2s_half *in_hi, const b2s_half *in_lo, int B, int Hin, int Win, int Cin,
                                 const b2s_half *w_hi, const b2s_half *w_lo, int kh, int kw, int stride, int pad,
                                 int Cout, int n_pad, const float *scale, const float *shift, int relu, int Hg, int Wg,
                                 void *out_hi, b2s_half *out_lo, int Hout, int Wout, int out_padded, int out_stride,
                                 int out_mul, int off_h, int off_w, const int *work_list, const int *work_count_dev,
                                 const int *bg_list, const int *bg_count_dev, const b2s_half *bg_hi,
                                 const b2s_half *bg_lo, int bg_margin, int list_rows, unsigned *status_dev,
                                 void *stream)
{
    return b2s_conv2d_tc_ex3(in_hi, in_lo, B, Hin, Win, Cin, w_hi, w_lo, kh, kw, stride, pad, Cout, n_pad, scale, shift,
                             relu, Hg, Wg, out_hi, out_lo, Hout, Wout, out_padded, out_stride, out_mul, off_h, off_w,
                             work_list, work_count_dev, bg_list, bg_count_dev, bg_hi, bg_lo, bg_margin, list_rows, 3, 0,
                             status_dev, stream);
}

// the same with the lists of b2s_rpn_block_plan (8x8 blocks)
extern "C" int b2s_conv2d_tc_ex(const b2s_half *in_hi, const b2s_half *in_lo, int B, int Hin, int Win, int Cin,
                                const b2s_half *w_hi, const b2s_half *w_lo, int kh, int kw, int stride, int pad,
                                int Cout, int n_pad, const float *scale, const float *shift, int relu, int Hg, int Wg,
                                void *out_hi, b2s_half *out_lo, int Hout, int Wout, int out_padded, int out_stride,
                                int out_mul, int off_h, int off_w, const int *work_list, const int *work_count_dev,
                                const int *bg_list, const int *bg_count_dev, const b2s_half *bg_hi,
                                const b2s_half *bg_lo, unsigned *status_dev, void *stream)
{
    return b2s_conv2d_tc_ex2(in_hi, in_lo, B, Hin, Win, Cin, w_hi, w_lo, kh, kw, stride, pad, Cout, n_pad, scale, shift,
                             relu, Hg, Wg, out_hi, out_lo, Hout, Wout, out_padded, out_stride, out_mul, off_h, off_w,
                             work_list, work_count_dev, bg_list, bg_count_dev, bg_hi, bg_lo, -1, 8, status_dev, stream);
}

// 3x3 pad 1 (taps = 9) or 1x1 (taps = 1), stride 1, output on the input grid
extern "C" int b2s_conv2d_tc(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin,
                             const b2s_half *w_hi, const b2s_half *w_lo, int taps, int Cout, int n_pad,
                             const float *scale, const float *shift, int relu, void *out_hi, b2s_half *out_lo,
                             int out_padded, int out_stride, unsigned *status_dev, void *stream_)
{
    B2S_REQUIRE(taps == 1 || taps == 9, "b2s_conv2d_tc: taps must be 1 or 9");
    const int k = taps == 9 ? 3 : 1;
    return b2s_conv2d_tc_ex(in_hi, in_lo, B, H, W, Cin, w_hi, w_lo, k, k, 1, taps == 9 ? 1 : 0, Cout, n_pad, scale, shift,
                            relu, H, W, out_hi, out_lo, H, W, out_padded, out_stride, 1, 0, 0, nullptr, nullptr, nullptr, nullptr,
                            nullptr, nullptr, status_dev, stream_);
}
