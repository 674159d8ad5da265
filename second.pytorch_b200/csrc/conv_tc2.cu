// conv_tc2.cu -- 3x3 RPN convolution with vertical activation reuse (wgmma, sm_90a).
//
// Why a second kernel: k_conv_tc (conv_tc.cu) loads a fresh [8 x 16 pixel, 64 channel] activation tile for every
// one of the 9 taps.  Here a stage is a 10-row x 16-col pixel tile (one 64-channel chunk, one horizontal tap offset
// dx), and the three vertical taps dy = 0,1,2 are the SAME stage viewed dy pixel rows (= 2048 B = two whole 1024-byte
// swizzle atoms) further down, so the wgmma descriptor just starts 2048*dy bytes later -- no swizzle-phase tricks.
// Activation bytes written to shared memory drop 2.4x against k_conv_tc.
//
// Work items are 16 x 16-pixel tiles (the granularity of the tile work list and of the background tiles, rpn_bg.cu);
// a work item is computed as two 8 x 16 halves, one after the other (the lower half only when it has image rows).
// A half is D[128 pixels, Cout = 128]: warpgroup g of the two consumer warpgroups owns pixel rows 4g .. 4g+3 of the
// half, 64 pixels x 128 channels of fp32 accumulators plus the same again for the running sum, which is what the
// register file holds at 384 threads per SM.
//
// Accumulation chains stay short (the tensor core's fp32 accumulate truncates: the rms error grows linearly with chain
// length): one chain = one (dx, chunk) group = 36 MMAs, added into fp32 registers with round-to-nearest adds.
//
// Warp roles (12 warps): 0 activation TMA producer, 3 weight TMA producer, 4-11 two consumer warpgroups (MMA,
// epilogue, background tiles).
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

using namespace b2s_tc;
constexpr int T2_H = 16, T2_W = 16;                 // work item: 256 output pixels
constexpr int HALF_H = 8;                           // rows computed at once (BLOCK_M = 128 pixels)
constexpr int HALO_H = HALF_H + 2;                  // rows of the activation stage
constexpr int kThreads2 = 384;
constexpr uint32_t X_PLANE_BYTES = HALO_H * T2_W * BLOCK_K * ELEM_BYTES;   // 20 KB (hi or lo)
constexpr uint32_t X_STAGE_BYTES = 2 * X_PLANE_BYTES;             // 40 KB
constexpr uint32_t W_PLANE_BYTES = 128 * BLOCK_K * ELEM_BYTES;             // 16 KB
// Weight ring of single planes: per dy the hi plane, then the lo plane.  Six slots = one whole (dx, chunk) group
// of weights in flight while the previous one is multiplied.
constexpr int X_STAGES = 2, W_STAGES = 6;
constexpr uint32_t DY_BYTES = T2_W * BLOCK_K * ELEM_BYTES;                 // one pixel row of the stage = 2048 B
static_assert(X_PLANE_BYTES % 1024 == 0, "stage planes are whole swizzle atoms");

struct Conv2Params {
    int B, H, W, Cin, Cout, relu;
    int tiles_h, tiles_w, num_tiles;
    const int *work_list, *work_count;   // optional (device): the tiles to compute, work_list[0 .. *work_count); tiles that
                                         // are not listed are "background" (b2s_rpn_bg_plan) and get their constant from
                                         // b2s_rpn_bg_fill.  NULL: every tile
    const int *bg_list, *bg_count;       // optional (device): background tiles of this layer's output; the consumer warps
    const __half *bg_hi, *bg_lo;         // copy them from the layer's empty-frame response bg_hi/bg_lo [H+2, W+2, Cout]
                                         // (one halo-padded frame) between their work items
    int out_stride;
    int dbg;                         // B2S_CONV2_DBG diagnostics (results wrong): 1 no activation loads, 2 no weight
                                     // loads, 4 no accumulator drain, 8 no global stores
    const float *scale, *shift;
    __half *out_hi, *out_lo;         // [B, H+2, W+2, out_stride] halo-padded fp16 planes (interior written)
    int *status;                     // bit B2S_STATUS_F16_RANGE raised when an activation exceeds the fp16 range
};

// number of work items and the i-th tile of this launch (dense: identity)
__device__ __forceinline__ int work_total(const Conv2Params &p) { return p.work_list ? min(*p.work_count, p.num_tiles) : p.num_tiles; }
__device__ __forceinline__ int work_tile(const Conv2Params &p, int i) { return p.work_list ? __ldg(&p.work_list[i]) : i; }
// 8-row halves of a tile that hold image rows (every role walks the same sequence)
__device__ __forceinline__ int halves_of(const Conv2Params &p, int tile)
{
    const int th = (tile / p.tiles_w) % p.tiles_h;
    return th * T2_H + HALF_H < p.H ? 2 : 1;
}

__global__ void __launch_bounds__(kThreads2, 1)
k_conv3x3_tc2(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
              const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
              const Conv2Params p)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *smem_x = smem;                                   // X_STAGES x 40 KB
    uint8_t *smem_w = smem + X_STAGES * X_STAGE_BYTES;        // W_STAGES x 16 KB
    __shared__ __align__(8) uint64_t bar_xfull[X_STAGES], bar_xempty[X_STAGES], bar_wfull[W_STAGES], bar_wempty[W_STAGES];
    __shared__ float s_scale[128], s_shift[128];

    const int warp = warp_idx_uniform(), lane = threadIdx.x & 31;
    const int kchunks = p.Cin / BLOCK_K;
    const int n_work = work_total(p);

    if (threadIdx.x < 128) {
        const int c = threadIdx.x;
        s_scale[c] = (p.scale && c < p.Cout) ? p.scale[c] : 1.f;
        s_shift[c] = (p.shift && c < p.Cout) ? p.shift[c] : 0.f;
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < X_STAGES; ++i) { mbar_init(&bar_xfull[i], 1); mbar_init(&bar_xempty[i], 8); }
        for (int i = 0; i < W_STAGES; ++i) { mbar_init(&bar_wfull[i], 1); mbar_init(&bar_wempty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 0) {
        // ===================== activation producer: one 10x16-pixel x 64-channel stage per (half, dx, chunk) ======
        if (lane == 0) {
            int xs = 0;
            uint32_t xph = 0;
            for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
                const int tile = work_tile(p, wi);
                const int tw = tile % p.tiles_w, th = (tile / p.tiles_w) % p.tiles_h, b = tile / (p.tiles_w * p.tiles_h);
                const int nh = halves_of(p, tile);
                for (int hf = 0; hf < nh; ++hf) {
                    const int h0 = th * T2_H + hf * HALF_H, w0 = tw * T2_W;
                    for (int dx = 0; dx < 3; ++dx)
                        for (int chunk = 0; chunk < kchunks; ++chunk) {
                            mbar_wait(&bar_xempty[xs], xph ^ 1);
                            uint8_t *st = smem_x + (size_t)xs * X_STAGE_BYTES;
                            if (p.dbg & 1) {                  // diagnostic: no activation loads (results wrong)
                                mbar_arrive(&bar_xfull[xs]);
                                if (++xs == X_STAGES) { xs = 0; xph ^= 1; }
                                continue;
                            }
                            mbar_arrive_expect_tx(&bar_xfull[xs], X_STAGE_BYTES);
                            // padded coordinates: output (h, w) reads padded rows h..h+2 and cols w..w+2
                            tma_load_4d(st, &map_x_hi, &bar_xfull[xs], chunk * BLOCK_K, w0 + dx, h0, b);
                            tma_load_4d(st + X_PLANE_BYTES, &map_x_lo, &bar_xfull[xs], chunk * BLOCK_K, w0 + dx, h0, b);
                            if (++xs == X_STAGES) { xs = 0; xph ^= 1; }
                        }
                }
            }
        }
    } else if (warp == 3) {
        // ===================== weight producer: W[tap = dy*3+dx][128, 64 ch] hi, then lo, per dy ===================
        if (lane == 0) {
            int ws = 0;
            uint32_t wph = 0;
            for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
                const int nh = halves_of(p, work_tile(p, wi));
                for (int hf = 0; hf < nh; ++hf)
                    for (int dx = 0; dx < 3; ++dx)
                        for (int chunk = 0; chunk < kchunks; ++chunk)
                            for (int dy = 0; dy < 3; ++dy)
                                for (int pl = 0; pl < 2; ++pl) {           // hi plane, then lo plane
                                    mbar_wait(&bar_wempty[ws], wph ^ 1);
                                    if (p.dbg & 2) {          // diagnostic: no weight loads (results wrong)
                                        mbar_arrive(&bar_wfull[ws]);
                                        if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
                                        continue;
                                    }
                                    mbar_arrive_expect_tx(&bar_wfull[ws], W_PLANE_BYTES);
                                    tma_load_3d(smem_w + (size_t)ws * W_PLANE_BYTES, pl ? &map_w_lo : &map_w_hi,
                                                &bar_wfull[ws], chunk * BLOCK_K, 0, dy * 3 + dx);
                                    if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
                                }
            }
        }
    } else if (warp >= 4) {
        // ===================== consumers: MMA + epilogue + background tiles =====================
        const int cg = (warp >> 2) - 1;             // warpgroup: pixel rows 4 cg .. 4 cg + 3 of the half
        const int wl = warp & 3;
        const uint32_t sx0 = smem_u32(smem_x), sw0 = smem_u32(smem_w);
        // Background tiles (csrc/rpn_bg.cu) of this layer's output: CTA c owns background tiles c, c + grid, ... and
        // spreads them over its work items.  One load / store instruction of the 256 consumer threads = one tile row of
        // one plane (16 pixels x 256 B, contiguous) of the layer's empty-frame response, which stays L2 resident.
        const int n_bg = p.bg_list ? min(*p.bg_count, p.num_tiles) : 0;
        const int my_bg = ((int)blockIdx.x < n_bg) ? (n_bg - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
        const int my_work = ((int)blockIdx.x < n_work) ? (n_work - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
        const int bg_quota = my_work > 0 ? (my_bg + my_work - 1) / my_work : my_bg;
        int bg_done = 0;
        const int e_tid = (warp - 4) * 32 + lane;                 // 0..255
        auto fill_bg = [&](int count) {
            const int chunk = e_tid & 15, px = e_tid >> 4;
            for (int q = 0; q < count && bg_done < my_bg; ++q, ++bg_done) {
                const int t = __ldg(&p.bg_list[(int)blockIdx.x + bg_done * (int)gridDim.x]);
                const int btw = t % p.tiles_w, bth = (t / p.tiles_w) % p.tiles_h, bb = t / (p.tiles_w * p.tiles_h);
                const int w = btw * T2_W + px;
                if (w >= p.W || chunk * 8 >= p.Cout) continue;
                const int rows = min(T2_H, p.H - bth * T2_H);
                const size_t fpix = (size_t)(bth * T2_H + 1) * (p.W + 2) + (w + 1);            // in the one-frame field
                const size_t opix = (size_t)bb * (p.H + 2) * (p.W + 2) + fpix;
                const uint4 *fh = reinterpret_cast<const uint4 *>(p.bg_hi + fpix * p.Cout + chunk * 8);
                const uint4 *fl = reinterpret_cast<const uint4 *>(p.bg_lo + fpix * p.Cout + chunk * 8);
                uint4 *oh = reinterpret_cast<uint4 *>(p.out_hi + opix * p.out_stride + chunk * 8);
                uint4 *ol = reinterpret_cast<uint4 *>(p.out_lo + opix * p.out_stride + chunk * 8);
                const size_t fstep = (size_t)(p.W + 2) * p.Cout / 8, ostep = (size_t)(p.W + 2) * p.out_stride / 8;
#pragma unroll 4
                for (int r = 0; r < rows; ++r) {
                    const uint4 vh = __ldg(fh + r * fstep), vl = __ldg(fl + r * fstep);
                    oh[r * ostep] = vh;
                    ol[r * ostep] = vl;
                }
            }
        };
        int xs = 0, ws = 0;
        uint32_t xph = 0, wph = 0;
        float sum[64], acc[64];
        for (int wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
            const int tile = work_tile(p, wi);
            const int tw = tile % p.tiles_w, th = (tile / p.tiles_w) % p.tiles_h, b = tile / (p.tiles_w * p.tiles_h);
            const int nh = halves_of(p, tile);
            for (int hf = 0; hf < nh; ++hf) {
#pragma unroll
                for (int j = 0; j < 64; ++j) sum[j] = 0.f;
                for (int g = 0; g < 3 * kchunks; ++g) {
                    mbar_wait(&bar_xfull[xs], xph);
                    const uint32_t sx = sx0 + (uint32_t)xs * X_STAGE_BYTES + (uint32_t)(cg * 4) * DY_BYTES;
#pragma unroll 1
                    for (int dy = 0; dy < 3; ++dy) {
                        int ws2 = ws + 1;
                        uint32_t wph2 = wph;
                        if (ws2 == W_STAGES) { ws2 = 0; wph2 ^= 1; }
                        mbar_wait(&bar_wfull[ws], wph);
                        mbar_wait(&bar_wfull[ws2], wph2);
                        const uint64_t x_hi = make_desc_sw128(sx + dy * DY_BYTES);
                        const uint64_t x_lo = make_desc_sw128(sx + X_PLANE_BYTES + dy * DY_BYTES);
                        const uint64_t w_hi = make_desc_sw128(sw0 + (uint32_t)ws * W_PLANE_BYTES);
                        const uint64_t w_lo = make_desc_sw128(sw0 + (uint32_t)ws2 * W_PLANE_BYTES);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);   // +32 B per K step
                            wgmma_ss<128>(acc, x_lo + koff, w_hi + koff, (dy | k) != 0);
                            wgmma_ss<128>(acc, x_hi + koff, w_hi + koff, 1);
                        }
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                            wgmma_ss<128>(acc, x_hi + koff, w_lo + koff, 1);
                        }
                        wgmma_commit();
                        wgmma_wait_all();
                        wgmma_fence_operands<64>(acc);
                        __syncwarp();
                        if (lane == 0) { mbar_arrive(&bar_wempty[ws]); mbar_arrive(&bar_wempty[ws2]); }
                        ws = ws2 + 1; wph = wph2;
                        if (ws == W_STAGES) { ws = 0; wph ^= 1; }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&bar_xempty[xs]);
                    if (++xs == X_STAGES) { xs = 0; xph ^= 1; }
                    if (!(p.dbg & 4)) {
#pragma unroll
                        for (int j = 0; j < 64; ++j) sum[j] = __fadd_rn(sum[j], acc[j]);
                    }
                }
                // BN scale/shift + ReLU + hi/lo fp16 split.  This thread holds pixels m0 = 16 wl + lane/4 and m0 + 8 of
                // the warpgroup's 64 (= rows 4 cg + m/16, column m % 16 of the half) and per 8-channel block j the
                // channel pair 8j + 2(lane % 4): one 4-byte store per plane, a quad of lanes writes 16 contiguous bytes.
                bool range_bad = false;
#pragma unroll
                for (int rh = 0; rh < 2; ++rh) {
                    const int m = wl * 16 + (lane >> 2) + rh * 8;
                    const int h = th * T2_H + hf * HALF_H + cg * 4 + m / T2_W, w = tw * T2_W + m % T2_W;
                    if (h >= p.H || w >= p.W || (p.dbg & 8)) continue;
                    const size_t pix = ((size_t)b * (p.H + 2) + (h + 1)) * (p.W + 2) + (w + 1);
                    __half *oh = p.out_hi + pix * p.out_stride, *ol = p.out_lo + pix * p.out_stride;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int c = 8 * j + 2 * (lane & 3);
                        if (c >= p.Cout) continue;                   // Cout is even (host check)
                        float x0 = fmaf(sum[4 * j + 2 * rh], s_scale[c], s_shift[c]);
                        float x1 = fmaf(sum[4 * j + 2 * rh + 1], s_scale[c + 1], s_shift[c + 1]);
                        if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                        range_bad |= (fabsf(x0) > 65504.f) | (fabsf(x1) > 65504.f);
                        const uint32_t p0 = split_f16(x0), p1 = split_f16(x1);
                        *reinterpret_cast<uint32_t *>(oh + c) = __byte_perm(p0, p1, 0x5410);
                        *reinterpret_cast<uint32_t *>(ol + c) = __byte_perm(p0, p1, 0x7632);
                    }
                }
                if (range_bad && p.status) atomicOr(p.status, B2S_STATUS_F16_RANGE);
            }
            fill_bg(bg_quota);
        }
        fill_bg(my_bg);                                          // whatever is left (a CTA without work items: all of it)
    }
}

}  // namespace

// called by b2s_conv2d_tc (conv_tc.cu) for taps == 9, n_pad == 128, halo-padded hi/lo output
int b2s_conv3x3_tc2(const __half *in_hi, const __half *in_lo, int B, int H, int W, int Cin, const __half *w_hi,
                    const __half *w_lo, int Cout, const float *scale, const float *shift, int relu, __half *out_hi,
                    __half *out_lo, int out_stride, const int *work_list, const int *work_count, const int *bg_list,
                    const int *bg_count, const __half *bg_hi, const __half *bg_lo, int *status, int num_sms,
                    cudaStream_t stream)
{
    using namespace b2s_tc;
    CUtensorMap x_hi, x_lo, m_w_hi, m_w_lo;
    {
        cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)(W + 2), (cuuint64_t)(H + 2), (cuuint64_t)B};
        cuuint64_t str[3] = {(cuuint64_t)Cin * ELEM_BYTES, (cuuint64_t)(W + 2) * Cin * ELEM_BYTES,
                             (cuuint64_t)(H + 2) * (W + 2) * Cin * ELEM_BYTES};
        cuuint32_t box[4] = {BLOCK_K, T2_W, HALO_H, 1};
        if (make_map(&x_hi, in_hi, 4, dims, str, box) || make_map(&x_lo, in_lo, 4, dims, str, box)) return -1;
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)Cin, 128, 9};
        cuuint64_t str[2] = {(cuuint64_t)Cin * ELEM_BYTES, (cuuint64_t)128 * Cin * ELEM_BYTES};
        cuuint32_t box[3] = {BLOCK_K, 128, 1};
        if (make_map(&m_w_hi, w_hi, 3, dims, str, box) || make_map(&m_w_lo, w_lo, 3, dims, str, box)) return -1;
    }
    Conv2Params p;
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.relu = relu;
    p.tiles_h = (H + T2_H - 1) / T2_H;
    p.tiles_w = (W + T2_W - 1) / T2_W;
    p.num_tiles = B * p.tiles_h * p.tiles_w;
    p.work_list = work_list; p.work_count = work_list ? work_count : nullptr;
    p.bg_list = bg_list; p.bg_count = bg_count; p.bg_hi = bg_hi; p.bg_lo = bg_lo;
    p.out_stride = out_stride;
    {
        static int dbg = -1;
        if (dbg < 0) { const char *e = getenv("B2S_CONV2_DBG"); dbg = e ? atoi(e) : 0; }
#ifdef B2S_DIAG
        p.dbg = dbg;            // diagnostics that corrupt results exist only in `make DIAG=1` builds
#else
        p.dbg = 0;
#endif
    }
    p.scale = scale; p.shift = shift; p.out_hi = out_hi; p.out_lo = out_lo; p.status = status;
    const size_t smem = (size_t)X_STAGES * X_STAGE_BYTES + (size_t)W_STAGES * W_PLANE_BYTES + 1024;
    B2S_SMEM_OPT_IN(k_conv3x3_tc2, smem);
    const int grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;     // (with a work list some CTAs may only fill)
    k_conv3x3_tc2<<<grid, kThreads2, smem, stream>>>(x_hi, x_lo, m_w_hi, m_w_lo, p);
    B2S_LAUNCH_OK();
    return 0;
}
