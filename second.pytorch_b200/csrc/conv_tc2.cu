// conv_tc2.cu -- 3x3 RPN convolution with vertical activation reuse (wgmma, sm_90a).
//
// Why a second kernel: k_conv_tc (conv_tc.cu) loads a fresh [8 x 16 pixel, 64 channel] activation tile for every
// one of the 9 taps.  Here a stage holds, per output strip, an (R+2)-row x 8-col pixel window (one 64-channel chunk,
// one horizontal tap offset dx), and the three vertical taps dy = 0,1,2 are the SAME window viewed dy pixel rows
// further down, so the wgmma descriptor just starts dy whole 1024-byte swizzle atoms later -- no swizzle-phase tricks.
//
// Output strips are 8 pixels wide and R = 8, 4 or 2 rows high (the granularity of the work list and of the background
// strips, rpn_bg.cu: 8 x 8 blocks of b2s_rpn_block_plan and of dense launches, 8 x R strips of b2s_rpn_strip_plan;
// the engine uses R = 4).  One consumer
// warpgroup's m64 accumulator tile is S = 8 / R strips.  An image row of 8 pixels x 64 fp16 channels is exactly one
// swizzle atom, and the window rows are interleaved in shared memory: window row r of strip s is atom r * S + s.  The
// A tile of tap dy is then the 8 contiguous atoms from dy * S on (stride 1024 B, as for one 8 x 8 block), and
// accumulator row m is strip s = (m / 8) % S, strip row (m / 8) / S, column m % 8.  R = 8 (S = 1) is one 10-row
// window per tile.
//
// A work item is a PAIR of warpgroup tiles: warpgroup g of pair i computes list entries S (2i + g) .. S (2i + g) + S - 1
// (dense: of all strips), D[64 pixels, Cout = 128]: 64 x 128 fp32 accumulators plus the same again for the running
// sum, which is what the register file holds at 384 threads per SM.  Both warpgroups multiply the same weight planes.
// Slots past the end of the list repeat the pair's first strip: they are computed and not stored.
//
// Accumulation chains stay short (the tensor core's fp32 accumulate truncates: the rms error grows linearly with chain
// length): one chain = one (dx, chunk) group = 36 MMAs, added into fp32 registers with round-to-nearest adds.  A
// pixel's sum does not depend on R or on which row of the tile it lands in, so every R gives the same bits.
//
// Warp roles (12 warps): 0 activation TMA producer, 1-2 background strips (the layer's empty-frame response: its
// constant interior value from registers, copied near the border; independently of the work items), 3 weight TMA
// producer, 4-11 two consumer warpgroups (MMA, epilogue).  The kernel is bound by the bytes it reads from L2, so the
// fill reading nothing for interior strips is worth as much as the MMAs it skips.
//
// P = products per K step: 3 (3xF16, above) or 1 (the f16 mode): one fp16 plane per operand, so a stage holds the hi
// windows only, the weight ring carries hi planes only (its six slots are then two whole (dx, chunk) groups), each K
// step is one wgmma, and the epilogue and the background fill write the hi plane only.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

using namespace b2s_tc;
constexpr int STRIP_W = 8;                          // output strip width: one image row of a strip = one swizzle atom
constexpr int kThreads2 = 384;
constexpr uint32_t ATOM_BYTES = STRIP_W * BLOCK_K * ELEM_BYTES;            // one pixel row of a window = 1024 B
constexpr uint32_t W_PLANE_BYTES = 128 * BLOCK_K * ELEM_BYTES;             // 16 KB
// Weight ring of single planes: per dy the hi plane, then the lo plane.  Six slots = one whole (dx, chunk) group
// of weights in flight while the previous one is multiplied.
constexpr int X_STAGES = 2, W_STAGES = 6;
static_assert(ATOM_BYTES == 1024, "window rows are whole swizzle atoms");

// shared-memory geometry for strips of R rows: S = 8 / R strips per warpgroup tile; P products per K step
template <int R, int P>
struct StripGeom {
    static_assert(R == 8 || R == 4 || R == 2, "strip heights 8, 4 and 2 are built");
    static_assert(P == 3 || P == 1, "products per K step: 3 (3xF16) or 1 (f16)");
    static constexpr int S = 8 / R;
    static constexpr int PLANES = P == 3 ? 2 : 1;                          // operand planes: hi, lo
    static constexpr uint32_t DY_BYTES = S * ATOM_BYTES;                    // one window row of all S strips
    static constexpr uint32_t X_TILE_BYTES = (R + 2) * DY_BYTES;           // one warpgroup tile's windows, one plane
    static constexpr uint32_t X_PLANE_BYTES = 2 * X_TILE_BYTES;            // hi or lo: both tiles of a pair
    static constexpr uint32_t X_STAGE_BYTES = PLANES * X_PLANE_BYTES;      // 3xF16, R = 8: 40 KB, R = 2: 64 KB
    static constexpr size_t SMEM_BYTES = (size_t)X_STAGES * X_STAGE_BYTES + (size_t)W_STAGES * W_PLANE_BYTES + 1024;
};

struct Conv2Params {
    int B, H, W, Cin, Cout, relu;
    int strips_h, strips_w, num_strips;  // strip id = (b * strips_h + sh) * strips_w + sw
    const int *work_list, *work_count;   // optional (device): the strips to compute, work_list[0 .. *work_count); strips
                                         // that are not listed are "background" (b2s_rpn_strip_plan) and get their
                                         // constant through bg_list.  NULL: every strip
    const int *bg_list, *bg_count;       // optional (device): background strips of this layer's output; warps 1-2 copy
    const __half *bg_hi, *bg_lo;         // them from the layer's empty-frame response bg_hi/bg_lo [H+2, W+2, Cout]
                                         // (one halo-padded frame)
    int bg_margin;                       // >= 0: the field equals its value at pixel (bg_margin, bg_margin) wherever it
                                         // is >= bg_margin pixels from every border; < 0: no such promise
    int out_stride;
    const float *scale, *shift;
    __half *out_hi, *out_lo;         // [B, H+2, W+2, out_stride] halo-padded fp16 planes (interior written)
    int *status;                     // bit B2S_STATUS_F16_RANGE raised when an activation exceeds the fp16 range
};

// number of listed strips and the i-th strip of this launch (dense: identity)
__device__ __forceinline__ int work_total(const Conv2Params &p) { return p.work_list ? min(*p.work_count, p.num_strips) : p.num_strips; }
__device__ __forceinline__ int work_strip(const Conv2Params &p, int i) { return p.work_list ? __ldg(&p.work_list[i]) : i; }

// first output pixel (h0, w0) and frame b of a strip
template <int R>
__device__ __forceinline__ void strip_origin(const Conv2Params &p, int id, int &h0, int &w0, int &b)
{
    w0 = (id % p.strips_w) * STRIP_W;
    h0 = ((id / p.strips_w) % p.strips_h) * R;
    b = id / (p.strips_w * p.strips_h);
}

template <int R, int P>
__global__ void __launch_bounds__(kThreads2, 1)
k_conv3x3_tc2(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
              const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
              const Conv2Params p)
{
    using G = StripGeom<R, P>;
    constexpr int S = G::S;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *smem_x = smem;                                   // X_STAGES x X_STAGE_BYTES
    uint8_t *smem_w = smem + X_STAGES * G::X_STAGE_BYTES;     // W_STAGES x 16 KB
    __shared__ __align__(8) uint64_t bar_xfull[X_STAGES], bar_xempty[X_STAGES], bar_wfull[W_STAGES], bar_wempty[W_STAGES];
    __shared__ float s_scale[128], s_shift[128];

    const int warp = warp_idx_uniform(), lane = threadIdx.x & 31;
    const int kchunks = p.Cin / BLOCK_K;
    const int n_work = work_total(p);
    const int n_pairs = (n_work + 2 * S - 1) / (2 * S);

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
        // ===================== activation producer: per (pair, dx, chunk) 2S windows of (R+2) x 8 pixels x 2 planes
        if (lane == 0) {
            int xs = 0;
            uint32_t xph = 0;
            for (int pi = blockIdx.x; pi < n_pairs; pi += gridDim.x) {
                int h0[2 * S], w0[2 * S], bb[2 * S];                  // slot j = g * S + s: strip s of warpgroup g
#pragma unroll
                for (int j = 0; j < 2 * S; ++j) {
                    const int e = 2 * S * pi + j;
                    strip_origin<R>(p, work_strip(p, e < n_work ? e : 2 * S * pi), h0[j], w0[j], bb[j]);   // tail: repeat
                }
                for (int dx = 0; dx < 3; ++dx)
                    for (int chunk = 0; chunk < kchunks; ++chunk) {
                        mbar_wait(&bar_xempty[xs], xph ^ 1);
                        uint8_t *st = smem_x + (size_t)xs * G::X_STAGE_BYTES;
                        mbar_arrive_expect_tx(&bar_xfull[xs], G::X_STAGE_BYTES);
                        // padded coordinates: output (h, w) reads padded rows h..h+2 and cols w..w+2; a box that
                        // reaches past the padded map (partial strips at the right / bottom edge) is zero-filled.
                        // Window row r of strip s goes to atom r * S + s: one (R+2)-row box when S = 1, else one
                        // single-row box per window row.
#pragma unroll
                        for (int j = 0; j < 2 * S; ++j) {
                            uint8_t *dst = st + (j / S) * G::X_TILE_BYTES + (j % S) * ATOM_BYTES;
                            const int x0 = w0[j] + dx;
#pragma unroll
                            for (int r = 0; r < (S == 1 ? 1 : R + 2); ++r) {
                                tma_load_4d(dst + r * G::DY_BYTES, &map_x_hi, &bar_xfull[xs], chunk * BLOCK_K, x0,
                                            h0[j] + r, bb[j]);
                                if constexpr (P == 3)
                                    tma_load_4d(dst + G::X_PLANE_BYTES + r * G::DY_BYTES, &map_x_lo, &bar_xfull[xs],
                                                chunk * BLOCK_K, x0, h0[j] + r, bb[j]);
                            }
                        }
                        if (++xs == X_STAGES) { xs = 0; xph ^= 1; }
                    }
            }
        }
    } else if (warp == 3) {
        // ===================== weight producer: W[tap = dy*3+dx][128, 64 ch] hi, then lo, per dy ===================
        if (lane == 0) {
            int ws = 0;
            uint32_t wph = 0;
            for (int pi = blockIdx.x; pi < n_pairs; pi += gridDim.x)
                for (int dx = 0; dx < 3; ++dx)
                    for (int chunk = 0; chunk < kchunks; ++chunk)
                        for (int dy = 0; dy < 3; ++dy)
                            for (int pl = 0; pl < G::PLANES; ++pl) {   // hi plane, then lo plane
                                mbar_wait(&bar_wempty[ws], wph ^ 1);
                                mbar_arrive_expect_tx(&bar_wfull[ws], W_PLANE_BYTES);
                                tma_load_3d(smem_w + (size_t)ws * W_PLANE_BYTES, pl ? &map_w_lo : &map_w_hi,
                                            &bar_wfull[ws], chunk * BLOCK_K, 0, dy * 3 + dx);
                                if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
                            }
        }
    } else if (warp <= 2) {
        // ===================== background strips (csrc/rpn_bg.cu): CTA c fills strips NF c .., NF (c + grid) .. of bg_list
        // Nothing in this launch reads the layer's output, so the fill needs no ordering against the MMA roles.  Thread
        // t copies the 16-byte channel chunk t % 16 of strip columns t / 16 and t / 16 + 4, all rows, both planes, from
        // the layer's empty-frame response (L2 resident); a warp moves two whole pixels (512 B) per instruction.  A
        // batch of U = NF strips x QL column halves is loaded before its first store: 16 loads in flight per thread.
        // Strips at least bg_margin pixels from every border get the field's interior value, which each thread holds
        // in registers: most background strips are stored without reading anything from L2.
        if (p.bg_list) {
            constexpr int NF = R >= 4 ? 1 : 2, QL = R >= 8 ? 1 : 2, U = NF * QL;
            const int n_bg = min(*p.bg_count, p.num_strips);
            const int t = (warp - 1) * 32 + lane;                     // 0..63
            const int chunk = t & 15, px = t >> 4;
            const int m = p.bg_margin;
            if (chunk * 8 < p.Cout) {
                const size_t fstep = (size_t)(p.W + 2) * p.Cout / 8, ostep = (size_t)(p.W + 2) * p.out_stride / 8;
                uint4 ch = make_uint4(0, 0, 0, 0), cl = ch;               // the interior value of this channel chunk
                if (m >= 0) {
                    const size_t cpix = (size_t)(m + 1) * (p.W + 2) + (m + 1);
                    ch = __ldg(reinterpret_cast<const uint4 *>(p.bg_hi + cpix * p.Cout + chunk * 8));
                    if constexpr (P == 3) cl = __ldg(reinterpret_cast<const uint4 *>(p.bg_lo + cpix * p.Cout + chunk * 8));
                }
                for (int i0 = blockIdx.x * NF; i0 < n_bg; i0 += gridDim.x * NF) {
#pragma unroll
                    for (int q0 = 0; q0 < 2; q0 += QL) {
                        uint4 vh[U][R], vl[U][R];
                        uint4 *oh[U], *ol[U];
                        int rows[U];                                   // rows of unit u to copy (0: none)
                        bool inner[U];                                 // unit u lies in the constant interior
#pragma unroll
                        for (int u = 0; u < U; ++u) {
                            const int i = i0 + u / QL;
                            int h0 = 0, w0 = 0, b = 0;
                            if (i < n_bg) strip_origin<R>(p, __ldg(&p.bg_list[i]), h0, w0, b);
                            const int w = w0 + px + 4 * (q0 + u % QL);
                            rows[u] = (i < n_bg && w < p.W) ? min(R, p.H - h0) : 0;
                            inner[u] = m >= 0 && h0 >= m && h0 + R <= p.H - m && w0 >= m && w0 + STRIP_W <= p.W - m;
                            const size_t fpix = (size_t)(h0 + 1) * (p.W + 2) + (w + 1);      // in the one-frame field
                            const size_t opix = (size_t)b * (p.H + 2) * (p.W + 2) + fpix;
                            const uint4 *fh = reinterpret_cast<const uint4 *>(p.bg_hi + fpix * p.Cout + chunk * 8);
                            const uint4 *fl = reinterpret_cast<const uint4 *>(p.bg_lo + fpix * p.Cout + chunk * 8);
                            oh[u] = reinterpret_cast<uint4 *>(p.out_hi + opix * p.out_stride + chunk * 8);
                            if constexpr (P == 3) {
                                ol[u] = reinterpret_cast<uint4 *>(p.out_lo + opix * p.out_stride + chunk * 8);
#pragma unroll
                                for (int r = 0; r < R; ++r)
                                    if (r < rows[u]) {
                                        if (inner[u]) { vh[u][r] = ch; vl[u][r] = cl; }
                                        else { vh[u][r] = __ldg(fh + r * fstep); vl[u][r] = __ldg(fl + r * fstep); }
                                    }
                            } else {
#pragma unroll
                                for (int r = 0; r < R; ++r)
                                    if (r < rows[u]) vh[u][r] = inner[u] ? ch : __ldg(fh + r * fstep);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < U; ++u)
#pragma unroll
                            for (int r = 0; r < R; ++r)
                                if (r < rows[u]) {
                                    if constexpr (P == 3) { oh[u][r * ostep] = vh[u][r]; ol[u][r * ostep] = vl[u][r]; }
                                    else oh[u][r * ostep] = vh[u][r];
                                }
                    }
                }
            }
        }
    } else {
        // ===================== consumers: MMA + epilogue =====================
        const int cg = (warp >> 2) - 1;             // warpgroup: list entries S (2i + cg) .. + S - 1 of pair i
        const int wl = warp & 3;
        const uint32_t sx0 = smem_u32(smem_x), sw0 = smem_u32(smem_w);
        int xs = 0, ws = 0;
        uint32_t xph = 0, wph = 0;
        float sum[64], acc[64];
        for (int pi = blockIdx.x; pi < n_pairs; pi += gridDim.x) {
#pragma unroll
            for (int j = 0; j < 64; ++j) sum[j] = 0.f;
            for (int g = 0; g < 3 * kchunks; ++g) {
                mbar_wait(&bar_xfull[xs], xph);
                const uint32_t sx = sx0 + (uint32_t)xs * G::X_STAGE_BYTES + (uint32_t)cg * G::X_TILE_BYTES;
#pragma unroll 1
                for (int dy = 0; dy < 3; ++dy) {
                    if constexpr (P == 1) {
                        mbar_wait(&bar_wfull[ws], wph);
                        const uint64_t x_hi = make_desc_sw128(sx + dy * G::DY_BYTES);
                        const uint64_t w_hi = make_desc_sw128(sw0 + (uint32_t)ws * W_PLANE_BYTES);
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                            wgmma_ss<128>(acc, x_hi + koff, w_hi + koff, (dy | k) != 0);
                        }
                        wgmma_commit();
                        wgmma_wait_all();
                        wgmma_fence_operands<64>(acc);
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&bar_wempty[ws]);
                        if (++ws == W_STAGES) { ws = 0; wph ^= 1; }
                        continue;
                    }
                    int ws2 = ws + 1;
                    uint32_t wph2 = wph;
                    if (ws2 == W_STAGES) { ws2 = 0; wph2 ^= 1; }
                    mbar_wait(&bar_wfull[ws], wph);
                    mbar_wait(&bar_wfull[ws2], wph2);
                    const uint64_t x_hi = make_desc_sw128(sx + dy * G::DY_BYTES);
                    const uint64_t x_lo = make_desc_sw128(sx + G::X_PLANE_BYTES + dy * G::DY_BYTES);
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
#pragma unroll
                for (int j = 0; j < 64; ++j) sum[j] = __fadd_rn(sum[j], acc[j]);
            }
            const int e0 = S * (2 * pi + cg);               // this warpgroup's first list entry
            if (e0 >= n_work) continue;                      // a repeat of the pair's first strip: nothing stored
            // BN scale/shift + ReLU + hi/lo fp16 split.  This thread holds accumulator rows m0 = 16 wl + lane/4 and
            // m0 + 8 of the warpgroup's 64 (atom m / 8 = 2 wl + rh = strip (m / 8) % S, strip row (m / 8) / S, column
            // m % 8 = lane / 4) and per 8-channel block j the channel pair 8j + 2(lane % 4): one 4-byte store per
            // plane, a quad of lanes writes 16 contiguous bytes.
            bool range_bad = false;
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int a = 2 * wl + rh;
                if (e0 + a % S >= n_work) continue;          // a repeated strip of a short tail
                int h0, w0, b;
                strip_origin<R>(p, work_strip(p, e0 + a % S), h0, w0, b);
                const int h = h0 + a / S, w = w0 + (lane >> 2);
                if (h >= p.H || w >= p.W) continue;
                const size_t pix = ((size_t)b * (p.H + 2) + (h + 1)) * (p.W + 2) + (w + 1);
                __half *oh = p.out_hi + pix * p.out_stride, *ol = P == 3 ? p.out_lo + pix * p.out_stride : nullptr;
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
                    if constexpr (P == 3) *reinterpret_cast<uint32_t *>(ol + c) = __byte_perm(p0, p1, 0x7632);
                }
            }
            if (range_bad && p.status) atomicOr(p.status, B2S_STATUS_F16_RANGE);
        }
    }
}

template <int R, int P>
int launch_tc2(const __half *in_hi, const __half *in_lo, const __half *w_hi, const __half *w_lo, Conv2Params &p,
               int num_sms, cudaStream_t stream)
{
    using G = StripGeom<R, P>;
    CUtensorMap x_hi, x_lo, m_w_hi, m_w_lo;
    {
        const int B = p.B, H = p.H, W = p.W, Cin = p.Cin;
        cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)(W + 2), (cuuint64_t)(H + 2), (cuuint64_t)B};
        cuuint64_t str[3] = {(cuuint64_t)Cin * ELEM_BYTES, (cuuint64_t)(W + 2) * Cin * ELEM_BYTES,
                             (cuuint64_t)(H + 2) * (W + 2) * Cin * ELEM_BYTES};
        // S = 1: a strip's whole (R+2)-row window is one box; else one box per window row (rows are interleaved)
        cuuint32_t box[4] = {BLOCK_K, STRIP_W, G::S == 1 ? (cuuint32_t)(R + 2) : 1u, 1};
        if (make_map(&x_hi, in_hi, 4, dims, str, box) || make_map(&x_lo, P == 3 ? in_lo : in_hi, 4, dims, str, box))
            return -1;
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)p.Cin, 128, 9};
        cuuint64_t str[2] = {(cuuint64_t)p.Cin * ELEM_BYTES, (cuuint64_t)128 * p.Cin * ELEM_BYTES};
        cuuint32_t box[3] = {BLOCK_K, 128, 1};
        if (make_map(&m_w_hi, w_hi, 3, dims, str, box) || make_map(&m_w_lo, P == 3 ? w_lo : w_hi, 3, dims, str, box))
            return -1;
    }
    p.strips_h = (p.H + R - 1) / R;
    p.strips_w = (p.W + STRIP_W - 1) / STRIP_W;
    p.num_strips = p.B * p.strips_h * p.strips_w;
    B2S_SMEM_OPT_IN((k_conv3x3_tc2<R, P>), G::SMEM_BYTES);
    const int max_pairs = (p.num_strips + 2 * G::S - 1) / (2 * G::S);
    const int grid = max_pairs < num_sms ? max_pairs : num_sms;     // (with a work list some CTAs may only fill)
    k_conv3x3_tc2<R, P><<<grid, kThreads2, G::SMEM_BYTES, stream>>>(x_hi, x_lo, m_w_hi, m_w_lo, p);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

// called by b2s_conv2d_tc_ex3 (conv_tc.cu) for taps == 9, n_pad == 128, halo-padded fp16 plane output; work_list /
// bg_list name 8 x list_rows strips (list_rows 8, 4 or 2); dense launches (no work list) run 8 x 8 blocks; products 3
// (hi/lo planes) or 1 (hi planes only)
int b2s_conv3x3_tc2(const __half *in_hi, const __half *in_lo, int B, int H, int W, int Cin, const __half *w_hi,
                    const __half *w_lo, int Cout, const float *scale, const float *shift, int relu, __half *out_hi,
                    __half *out_lo, int out_stride, const int *work_list, const int *work_count, const int *bg_list,
                    const int *bg_count, const __half *bg_hi, const __half *bg_lo, int bg_margin, int list_rows,
                    int products, int *status, int num_sms, cudaStream_t stream)
{
    Conv2Params p;
    p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.relu = relu;
    p.work_list = work_list; p.work_count = work_list ? work_count : nullptr;
    p.bg_list = bg_list; p.bg_count = bg_count; p.bg_hi = bg_hi; p.bg_lo = bg_lo;
    p.bg_margin = (bg_list && bg_margin >= 0 && 2 * bg_margin < H && 2 * bg_margin < W) ? bg_margin : -1;
    p.out_stride = out_stride;
    p.scale = scale; p.shift = shift; p.out_hi = out_hi; p.out_lo = out_lo; p.status = status;
    if (products == 1) {
        if (work_list && list_rows == 2) return launch_tc2<2, 1>(in_hi, in_lo, w_hi, w_lo, p, num_sms, stream);
        if (work_list && list_rows == 4) return launch_tc2<4, 1>(in_hi, in_lo, w_hi, w_lo, p, num_sms, stream);
        return launch_tc2<8, 1>(in_hi, in_lo, w_hi, w_lo, p, num_sms, stream);
    }
    if (work_list && list_rows == 2) return launch_tc2<2, 3>(in_hi, in_lo, w_hi, w_lo, p, num_sms, stream);
    if (work_list && list_rows == 4) return launch_tc2<4, 3>(in_hi, in_lo, w_hi, w_lo, p, num_sms, stream);
    return launch_tc2<8, 3>(in_hi, in_lo, w_hi, w_lo, p, num_sms, stream);
}
