// rpn_tail.cu -- the tail of a single-scale RPNV2 in ONE kernel (b2s_rpn_tail_tc):
//     y     = relu(bn(deblock(x)))            ConvTranspose2d k = s = 1  ==  1x1 conv, 128 -> 128   (rpn.py:264-299)
//     heads = [conv_box | conv_cls | conv_dir_cls](y)   1x1, 128 -> <= 32 packed channels + bias  (rpn.py:386-420)
// car.fhd / all.fhd: layer_nums [5], upsample_strides [1], num_upsample_filters [128].
//
// As two b2s_conv2d_tc launches y makes a round trip through HBM (2 x 577 MB at 32 frames).  Here y never leaves the
// SM: GEMM 1 accumulates it in the registers of the consumer warpgroup, BN + ReLU + the hi/lo split run on those
// registers, and the packed fp16 pairs are directly the A operand of GEMM 2 (wgmma with A from registers: the
// accumulator fragment of a 16-column block pair IS the A fragment of a 16-wide K step, no shuffle needed).  Per
// 128-pixel tile the kernel reads 64 KB of x and writes 16 KB of head records, instead of 208 KB of traffic.  Both
// weight sets (80 KB as hi/lo planes) stay resident in shared memory and the rest of it is a 4-slot x ring (two tiles
// in flight).  The MMA sequences, the epilogue arithmetic and the 3xF16 split are exactly those of k_conv_tc
// (conv_tc.cu) for the two layers, so the records are BIT-IDENTICAL to the two-launch path (tested).
//
// CTA = 3 warpgroups, persistent over 8 x 16-pixel tiles:
//   warp 0            TMA: weights once, then per tile the two 64-channel K blocks of x (hi + lo) into the ring
//   warps 1-3         background tiles (b2s_rpn_tail_tc_ex with a background list): their records are the records of
//                     an empty frame (the tail run once on the last layer's empty-frame response), stored from a
//                     record each thread holds in registers where the tile lies >= margin pixels from every border,
//                     copied from that one-frame record field nearer to it.  Nothing in the launch reads the records.
//   warpgroups 1, 2   consumers: warpgroup g owns tile pixels 64g .. 64g+63 through GEMM 1, the y epilogue, GEMM 2
//                     and the record stores
// With a work list, TMA and consumers walk the listed tiles only (a tile id = (b * tiles_h + th) * tiles_w + tw).
//
// P = products per K step: 3 (3xF16, above) or 1 (the f16 mode): x and both weight sets are single fp16 planes (half
// the shared memory), GEMM 1 is one wgmma per K step, y is rounded to one fp16 plane, and GEMM 2 is one register-A
// wgmma per K step.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

using namespace b2s_tc;
constexpr int TILE_H = 8, TILE_W = 16;    // BLOCK_M = 128 pixels
constexpr int C = 128;                    // channels of x and y
constexpr int KB = C / BLOCK_K;           // 2 K blocks of 64 channels
constexpr int N1 = 128;                   // GEMM 1 N (= channels of y)
constexpr int N2 = 32;                    // GEMM 2 N (packed head channels, zero padded)
constexpr int kThreads = 384;             // 1 producer warpgroup + 2 consumer warpgroups
constexpr int XS = 2 * KB;                // x ring slots (one K block of one tile each)

// shared-memory layout for P products per K step (PL = 2 planes for 3xF16, 1 for f16)
template <int P>
struct TailGeom {
    static_assert(P == 3 || P == 1, "products per K step: 3 (3xF16) or 1 (f16)");
    static constexpr int PL = P == 3 ? 2 : 1;
    static constexpr uint32_t W1_KB_BYTES = PL * N1 * BLOCK_K * ELEM_BYTES;   // hi + lo of one K block: 32 KB
    static constexpr uint32_t W2_KB_BYTES = PL * N2 * BLOCK_K * ELEM_BYTES;   // ... of the head weights: 8 KB
    static constexpr uint32_t X_STAGE_BYTES = PL * A_TILE_BYTES;              // hi + lo of one K block of x: 32 KB
    static constexpr uint32_t OFF_W1 = 0, OFF_W2 = OFF_W1 + KB * W1_KB_BYTES, OFF_X = OFF_W2 + KB * W2_KB_BYTES;
    static constexpr size_t SMEM_BYTES = OFF_X + XS * X_STAGE_BYTES + 1024;
    static_assert((OFF_W2 % 1024) == 0 && (OFF_X % 1024) == 0 && (N2 * BLOCK_K * ELEM_BYTES) % 1024 == 0,
                  "operand tiles are 1024-byte aligned (SWIZZLE_128B)");
};

struct TailParams {
    int B, H, W, tiles_h, tiles_w, num_tiles;
    int cout2, out_stride;
    const float *scale1, *shift1, *scale2, *shift2;
    float *out;
    int *status;
    const int *work_list, *work_count;   // optional (device): the tiles to compute; NULL: every tile
    const int *bg_list, *bg_count;       // optional (device): tiles whose records come from `field`
    const float *field;                  // [H, W, out_stride]: the records of an empty frame
    int margin;                          // >= 0: field equals its record at (margin, margin) wherever it is >= margin
                                         // pixels from every border; < 0: no such promise
};

template <int P>
__global__ void __launch_bounds__(kThreads, 1)
k_rpn_tail(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
           const __grid_constant__ CUtensorMap map_w1_hi, const __grid_constant__ CUtensorMap map_w1_lo,
           const __grid_constant__ CUtensorMap map_w2_hi, const __grid_constant__ CUtensorMap map_w2_lo,
           const TailParams p)
{
    using G = TailGeom<P>;
    constexpr uint32_t W1_KB_BYTES = G::W1_KB_BYTES, W2_KB_BYTES = G::W2_KB_BYTES, X_STAGE_BYTES = G::X_STAGE_BYTES;
    constexpr uint32_t OFF_W1 = G::OFF_W1, OFF_W2 = G::OFF_W2, OFF_X = G::OFF_X;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t bar_w, bar_xfull[XS], bar_xempty[XS];
    __shared__ float s_scale1[N1], s_shift1[N1], s_scale2[N2], s_shift2[N2];

    const int warp = warp_idx_uniform(), lane = threadIdx.x & 31;
    if (threadIdx.x < N1) {
        s_scale1[threadIdx.x] = p.scale1 ? p.scale1[threadIdx.x] : 1.f;
        s_shift1[threadIdx.x] = p.shift1 ? p.shift1[threadIdx.x] : 0.f;
    }
    if (threadIdx.x < N2) {
        const int c = threadIdx.x;
        s_scale2[c] = (p.scale2 && c < p.cout2) ? p.scale2[c] : 1.f;
        s_shift2[c] = (p.shift2 && c < p.cout2) ? p.shift2[c] : 0.f;
    }
    if (warp == 1 && lane == 0) {
        mbar_init(&bar_w, 1);
        for (int i = 0; i < XS; ++i) { mbar_init(&bar_xfull[i], 1); mbar_init(&bar_xempty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int n_work = p.work_list ? min(*p.work_count, p.num_tiles) : p.num_tiles;
    const auto tile_at = [&](int i) { return p.work_list ? __ldg(&p.work_list[i]) : i; };
    const bool has_work = (int)blockIdx.x < n_work;

    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0 && has_work) {
            mbar_arrive_expect_tx(&bar_w, KB * (W1_KB_BYTES + W2_KB_BYTES));
            for (int kb = 0; kb < KB; ++kb) {
                tma_load_3d(smem + OFF_W1 + kb * W1_KB_BYTES, &map_w1_hi, &bar_w, kb * BLOCK_K, 0, 0);
                if constexpr (P == 3)
                    tma_load_3d(smem + OFF_W1 + kb * W1_KB_BYTES + W1_KB_BYTES / 2, &map_w1_lo, &bar_w, kb * BLOCK_K, 0, 0);
                tma_load_3d(smem + OFF_W2 + kb * W2_KB_BYTES, &map_w2_hi, &bar_w, kb * BLOCK_K, 0, 0);
                if constexpr (P == 3)
                    tma_load_3d(smem + OFF_W2 + kb * W2_KB_BYTES + W2_KB_BYTES / 2, &map_w2_lo, &bar_w, kb * BLOCK_K, 0, 0);
            }
            int u = 0;                                                 // K blocks of x loaded so far: slot u % XS, its (u / XS)-th use
            for (int i = blockIdx.x; i < n_work; i += gridDim.x) {
                const int tile = tile_at(i);
                const int tw = tile % p.tiles_w, th = (tile / p.tiles_w) % p.tiles_h, b = tile / (p.tiles_w * p.tiles_h);
                const int h0 = th * TILE_H + 1, w0 = tw * TILE_W + 1;          // + 1: the one-pixel halo of the input planes
                for (int kb = 0; kb < KB; ++kb, ++u) {
                    const int slot = u % XS;
                    mbar_wait(&bar_xempty[slot], (uint32_t)((u / XS) & 1) ^ 1u);
                    uint8_t *st = smem + OFF_X + slot * X_STAGE_BYTES;
                    mbar_arrive_expect_tx(&bar_xfull[slot], X_STAGE_BYTES);
                    tma_load_4d(st, &map_x_hi, &bar_xfull[slot], kb * BLOCK_K, w0, h0, b);
                    if constexpr (P == 3) tma_load_4d(st + A_TILE_BYTES, &map_x_lo, &bar_xfull[slot], kb * BLOCK_K, w0, h0, b);
                }
            }
        }
    } else if (warp <= 3) {
        // ===================== background tiles: thread t stores the 16-byte record chunk q = t % nq of pixels
        // t / nq, t / nq + per, ... of each tile (per = 96 / nq pixels per pass)
        const int nq = p.cout2 / 4, per = 96 / nq;
        const int t = (warp - 1) * 32 + lane, q = t % nq;
        const size_t s4 = (size_t)p.out_stride / 4;
        if (p.bg_list && t < per * nq) {
            const int n_bg = min(*p.bg_count, p.num_tiles);
            const int m = p.margin;
            const float4 *field = reinterpret_cast<const float4 *>(p.field);
            float4 *out = reinterpret_cast<float4 *>(p.out);
            const float4 c = m >= 0 ? __ldg(field + ((size_t)m * p.W + m) * s4 + q) : make_float4(0.f, 0.f, 0.f, 0.f);
            for (int i = blockIdx.x; i < n_bg; i += gridDim.x) {
                const int tile = __ldg(&p.bg_list[i]);
                const int tw = tile % p.tiles_w, th = (tile / p.tiles_w) % p.tiles_h, b = tile / (p.tiles_w * p.tiles_h);
                const int h0 = th * TILE_H, w0 = tw * TILE_W;
                const bool inner = m >= 0 && h0 >= m && h0 + TILE_H <= p.H - m && w0 >= m && w0 + TILE_W <= p.W - m;
                for (int px = t / nq; px < TILE_H * TILE_W; px += per) {
                    const int h = h0 + px / TILE_W, w = w0 + px % TILE_W;
                    if (h >= p.H || w >= p.W) continue;
                    const size_t f = (size_t)h * p.W + w;
                    out[((size_t)b * p.H * p.W + f) * s4 + q] = inner ? c : __ldg(field + f * s4 + q);
                }
            }
        }
    } else {
        // ===================== consumers =====================
        const int cg = (warp >> 2) - 1;                          // tile pixels 64 cg .. 64 cg + 63
        const int wl = warp & 3;
        const uint32_t smem0 = smem_u32(smem);
        const uint32_t a_off = (uint32_t)cg * 64u * 128u;
        bool range_bad = false;
        if (has_work) mbar_wait(&bar_w, 0);
        int u = 0;
        for (int i = blockIdx.x; i < n_work; i += gridDim.x) {
            const int tile = tile_at(i);
            const int tw = tile % p.tiles_w, th = (tile / p.tiles_w) % p.tiles_h, b = tile / (p.tiles_w * p.tiles_h);
            // ---- GEMM 1: D1 = x * W1^T; per K step the three products of the 3xF16 split in k_conv_tc's order
            float d1[N1 / 2];
            for (int kb = 0; kb < KB; ++kb) {
                const int slot = (u + kb) % XS;
                mbar_wait(&bar_xfull[slot], (uint32_t)(((u + kb) / XS) & 1));
                const uint32_t xa = smem0 + OFF_X + slot * X_STAGE_BYTES + a_off;
                const uint32_t wb = smem0 + OFF_W1 + kb * W1_KB_BYTES;
                const uint64_t a_hi = make_desc_sw128(xa), b_hi = make_desc_sw128(wb);
                wgmma_fence();
                if constexpr (P == 3) {
                    const uint64_t a_lo = make_desc_sw128(xa + A_TILE_BYTES), b_lo = make_desc_sw128(wb + W1_KB_BYTES / 2);
#pragma unroll
                    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
                        const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                        wgmma_ss<N1>(d1, a_lo + koff, b_hi + koff, (kb | k) != 0);
                        wgmma_ss<N1>(d1, a_hi + koff, b_lo + koff, 1);
                        wgmma_ss<N1>(d1, a_hi + koff, b_hi + koff, 1);
                    }
                } else {
#pragma unroll
                    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
                        const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                        wgmma_ss<N1>(d1, a_hi + koff, b_hi + koff, (kb | k) != 0);
                    }
                }
                wgmma_commit();
            }
            wgmma_wait_all();
            wgmma_fence_operands<N1 / 2>(d1);
            __syncwarp();
            if (lane == 0)
                for (int kb = 0; kb < KB; ++kb) mbar_arrive(&bar_xempty[(u + kb) % XS]);
            u += KB;
            // ---- y = relu(D1 * scale1 + shift1) -> fp16 hi/lo pairs = the A fragments of GEMM 2.  K step s covers
            // channels 16s .. 16s+15 = accumulator blocks 2s, 2s+1: a[0] = block 2s row r, a[1] = block 2s row r+8,
            // a[2] / a[3] = block 2s+1 rows r / r+8.
            uint32_t yh[N1 / 4], yl[N1 / 4];
#pragma unroll
            for (int i = 0; i < N1 / 4; ++i) {
                const int blk = i >> 1;                            // 8-column block of register pair i
                const int c = 8 * blk + 2 * (lane & 3);
                float x0 = fmaf(__fadd_rn(0.f, d1[2 * i]), s_scale1[c], s_shift1[c]);
                float x1 = fmaf(__fadd_rn(0.f, d1[2 * i + 1]), s_scale1[c + 1], s_shift1[c + 1]);
                x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f);
                range_bad |= (fabsf(x0) > 65504.f) | (fabsf(x1) > 65504.f);
                const uint32_t p0 = split_f16(x0), p1 = split_f16(x1);
                yh[i] = __byte_perm(p0, p1, 0x5410);
                if constexpr (P == 3) yl[i] = __byte_perm(p0, p1, 0x7632);
            }
            // ---- GEMM 2: D2 = y * W2^T (A from registers)
            float d2[N2 / 2];
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < C / MMA_K; ++s) {
                const int kb = s / (BLOCK_K / MMA_K), k = s % (BLOCK_K / MMA_K);
                const uint32_t wb = smem0 + OFF_W2 + kb * W2_KB_BYTES;
                const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                const uint64_t b_hi = make_desc_sw128(wb) + koff;
                if constexpr (P == 3) {
                    const uint64_t b_lo = make_desc_sw128(wb + W2_KB_BYTES / 2) + koff;
                    wgmma_rs<N2>(d2, &yl[4 * s], b_hi, s != 0);
                    wgmma_rs<N2>(d2, &yh[4 * s], b_lo, 1);
                    wgmma_rs<N2>(d2, &yh[4 * s], b_hi, 1);
                } else {
                    wgmma_rs<N2>(d2, &yh[4 * s], b_hi, s != 0);
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            wgmma_fence_operands<N2 / 2>(d2);
            // ---- records = D2 * scale2 + shift2 (bias) -> fp32 [B, H, W, out_stride]
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int m = cg * 64 + wl * 16 + (lane >> 2) + rh * 8;
                const int hh = th * TILE_H + m / TILE_W, ww = tw * TILE_W + m % TILE_W;
                if (hh >= p.H || ww >= p.W) continue;
                float *outp = p.out + (((size_t)b * p.H + hh) * p.W + ww) * p.out_stride;
#pragma unroll
                for (int j = 0; j < N2 / 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    if (c >= p.cout2) continue;                  // cout2 is a multiple of 4
                    const float v0 = fmaf(__fadd_rn(0.f, d2[4 * j + 2 * rh]), s_scale2[c], s_shift2[c]);
                    const float v1 = fmaf(__fadd_rn(0.f, d2[4 * j + 2 * rh + 1]), s_scale2[c + 1], s_shift2[c + 1]);
                    *reinterpret_cast<float2 *>(outp + c) = make_float2(v0, v1);
                }
            }
        }
        if (__any_sync(0xffffffffu, range_bad) && lane == 0 && p.status) atomicOr(p.status, B2S_STATUS_F16_RANGE);
    }
}

}  // namespace

// in: halo-padded hi/lo planes [B, H+2, W+2, 128]; w1: [128][128] (y channel, x channel), w2: [n_pad][128] (rows >= cout2
// zero), both K-major hi/lo planes pre-scaled by a power of two folded into scale1 / scale2; out: fp32 [B, H, W, out_stride].
// products = 3: 3xF16; products = 1: the f16 mode, in_lo, w1_lo and w2_lo must be NULL.
extern "C" int b2s_rpn_tail_tc_ex2(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin,
                                   const b2s_half *w1_hi, const b2s_half *w1_lo, int Cmid, const float *scale1,
                                   const float *shift1, const b2s_half *w2_hi, const b2s_half *w2_lo, int cout2,
                                   int n_pad2, const float *scale2, const float *shift2, float *out, int out_stride,
                                   const int *work_list, const int *work_count, const int *bg_list, const int *bg_count,
                                   const float *field, int margin, int products, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && in_lo == nullptr && w1_lo == nullptr && w2_lo == nullptr),
                "b2s_rpn_tail_tc: products must be 3 (3xF16) or 1 (f16, no lo planes)");
    const bool three = products == 3;
    B2S_REQUIRE(Cin == C && Cmid == N1, "b2s_rpn_tail_tc: built for a 128 -> 128 deblock (got %d -> %d)", Cin, Cmid);
    B2S_REQUIRE(n_pad2 == N2 && cout2 >= 4 && cout2 <= n_pad2 && cout2 % 4 == 0 && out_stride >= cout2 && out_stride % 4 == 0,
                "b2s_rpn_tail_tc: up to 32 packed head channels (multiple of 4), out_stride a multiple of 4");
    B2S_REQUIRE(B >= 1 && H >= 1 && W >= 1 && ((uintptr_t)out & 15) == 0, "b2s_rpn_tail_tc: bad sizes / unaligned output");
    B2S_REQUIRE((work_list == nullptr) == (work_count == nullptr) && (bg_list == nullptr) == (bg_count == nullptr) &&
                    (bg_list == nullptr || (field != nullptr && ((uintptr_t)field & 15) == 0)),
                "b2s_rpn_tail_tc_ex: a list needs its count, a background list a 16-byte aligned record field");
    CUtensorMap x_hi, x_lo, m1_hi, m1_lo, m2_hi, m2_lo;
    {
        cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)(W + 2), (cuuint64_t)(H + 2), (cuuint64_t)B};
        cuuint64_t str[3] = {(cuuint64_t)C * ELEM_BYTES, (cuuint64_t)(W + 2) * C * ELEM_BYTES,
                             (cuuint64_t)(H + 2) * (W + 2) * C * ELEM_BYTES};
        cuuint32_t box[4] = {BLOCK_K, TILE_W, TILE_H, 1};
        if (make_map(&x_hi, in_hi, 4, dims, str, box) || (three && make_map(&x_lo, in_lo, 4, dims, str, box))) return -1;
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)N1, 1};
        cuuint64_t str[2] = {(cuuint64_t)C * ELEM_BYTES, (cuuint64_t)N1 * C * ELEM_BYTES};
        cuuint32_t box[3] = {BLOCK_K, N1, 1};
        if (make_map(&m1_hi, w1_hi, 3, dims, str, box) || (three && make_map(&m1_lo, w1_lo, 3, dims, str, box)))
            return -1;
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)n_pad2, 1};
        cuuint64_t str[2] = {(cuuint64_t)C * ELEM_BYTES, (cuuint64_t)n_pad2 * C * ELEM_BYTES};
        cuuint32_t box[3] = {BLOCK_K, (cuuint32_t)n_pad2, 1};
        if (make_map(&m2_hi, w2_hi, 3, dims, str, box) || (three && make_map(&m2_lo, w2_lo, 3, dims, str, box)))
            return -1;
    }
    TailParams p;
    p.B = B; p.H = H; p.W = W;
    p.tiles_h = (H + TILE_H - 1) / TILE_H;
    p.tiles_w = (W + TILE_W - 1) / TILE_W;
    p.num_tiles = B * p.tiles_h * p.tiles_w;
    p.cout2 = cout2; p.out_stride = out_stride;
    p.scale1 = scale1; p.shift1 = shift1; p.scale2 = scale2; p.shift2 = shift2;
    p.out = out; p.status = (int *)status_dev;
    p.work_list = work_list; p.work_count = work_count; p.bg_list = bg_list; p.bg_count = bg_count; p.field = field;
    p.margin = (bg_list && margin >= 0 && 2 * margin < H && 2 * margin < W) ? margin : -1;
    const int num_sms = num_sms_current();
    const int grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
    if (three) {
        B2S_SMEM_OPT_IN(k_rpn_tail<3>, TailGeom<3>::SMEM_BYTES);
        k_rpn_tail<3><<<grid, kThreads, TailGeom<3>::SMEM_BYTES, stream>>>(x_hi, x_lo, m1_hi, m1_lo, m2_hi, m2_lo, p);
    } else {
        B2S_SMEM_OPT_IN(k_rpn_tail<1>, TailGeom<1>::SMEM_BYTES);
        k_rpn_tail<1><<<grid, kThreads, TailGeom<1>::SMEM_BYTES, stream>>>(x_hi, x_hi, m1_hi, m1_hi, m2_hi, m2_hi, p);
    }
    B2S_LAUNCH_OK();
    return 0;
}

// the 3xF16 form
extern "C" int b2s_rpn_tail_tc_ex(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin,
                                  const b2s_half *w1_hi, const b2s_half *w1_lo, int Cmid, const float *scale1,
                                  const float *shift1, const b2s_half *w2_hi, const b2s_half *w2_lo, int cout2,
                                  int n_pad2, const float *scale2, const float *shift2, float *out, int out_stride,
                                  const int *work_list, const int *work_count, const int *bg_list, const int *bg_count,
                                  const float *field, int margin, unsigned *status_dev, void *stream)
{
    return b2s_rpn_tail_tc_ex2(in_hi, in_lo, B, H, W, Cin, w1_hi, w1_lo, Cmid, scale1, shift1, w2_hi, w2_lo, cout2, n_pad2,
                               scale2, shift2, out, out_stride, work_list, work_count, bg_list, bg_count, field, margin, 3,
                               status_dev, stream);
}

extern "C" int b2s_rpn_tail_tc(const b2s_half *in_hi, const b2s_half *in_lo, int B, int H, int W, int Cin,
                               const b2s_half *w1_hi, const b2s_half *w1_lo, int Cmid, const float *scale1,
                               const float *shift1, const b2s_half *w2_hi, const b2s_half *w2_lo, int cout2, int n_pad2,
                               const float *scale2, const float *shift2, float *out, int out_stride, unsigned *status_dev,
                               void *stream)
{
    return b2s_rpn_tail_tc_ex(in_hi, in_lo, B, H, W, Cin, w1_hi, w1_lo, Cmid, scale1, shift1, w2_hi, w2_lo, cout2, n_pad2,
                              scale2, shift2, out, out_stride, nullptr, nullptr, nullptr, nullptr, nullptr, -1,
                              status_dev, stream);
}
