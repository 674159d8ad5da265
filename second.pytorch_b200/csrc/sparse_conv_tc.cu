// sparse_conv_tc.cu -- sparse convolution inner product on the tensor pipe (b2s_sparse_conv_tc, b2s_sparse_conv_tc_plan).
//
// Output-stationary like sparse_conv.cu (one CTA owns 128 output rows at a time; nbr[o][k] names the input row feeding
// output row o through kernel offset k), but the per-offset product
//     D[128 rows, Cout] += A[128 gathered rows, 64 channels] * W[k][Cout, 64 channels]^T
// is a wgmma (f16 -> f32) on the 3xF16 hi/lo split (tc_common.cuh), accumulating in registers.
//
// K block = one 128-byte-wide slice of the reduction (64 fp16 channels) = PACK = 64/Cin consecutive kernel offsets
// side by side (Cin = 64: one offset; 32: 2; 16: 4; 8: 8; the weights arrive pre-packed as [K block][Cout][64], see
// b2second/tc.py: pack_sparse_weights; a 3- or 4-feature input layer is zero-padded to 8 channels).
//
// Tile plan (sparse_plan.cu): tile_mask[tile] says which kernel offsets ANY of the tile's 128 rows needs; a K block
// none of whose offsets is needed is skipped by every role (weights not loaded, rows not gathered, MMAs not issued).
// perm[] (optional) makes a tile = 128 rows with a similar neighbourhood shape, which roughly halves the K blocks of the
// SECOND middle encoder.  A missing neighbour contributes exact zeros and the accumulation chains have FIXED K-block
// boundaries (chain c = K blocks [c*CHAIN_KB, (c+1)*CHAIN_KB)), so the value of an output row does not depend on which
// rows share its tile: planned and unplanned results are bit-identical.
//
// Warp roles (16 warps):
//   warps 0-7   gather producers.  Gather warp w OWNS pipeline stage w % 4 and the tile's row half w / 4: it handles
//               every 4th K block, all 16-byte cp.async copies of its 64 rows (hi and lo planes) into the K-major
//               SWIZZLE_128B A tile, zero-fill for missing neighbours, completion signalled on the stage's mbarrier
//               with cp.async.mbarrier.arrive.noinc.  The neighbour-table entries of the NEXT owned K block are
//               loaded (straight from global / L1) before the current one is waited for.  Lane 0 of the row-half-0
//               warp of a K block also issues its weight tile (bulk tensor load, SWIZZLE_128B) once the stage is free.
//   warps 8-15  two consumer warpgroups: warpgroup g issues the wgmmas of tile rows 64g .. 64g+63 and owns their
//               accumulators; per-chain partial sums go into fp32 running sums with round-to-nearest adds (the tensor
//               core's own accumulate is not RN -- see conv_tc.cu), then BN scale/shift + ReLU, hi/lo split, stores.
//               Consumers only wait on full stages and release them: a consumer warp that also issued the weights
//               would wait for the OTHER warpgroup to release each stage, tying the two together on every K block
//               (that cost 25-35 % of the time of every layer but the last, 3x1x1 one, on H100).
//
// P = products per K block: 3 (3xF16, above) or 1 (the f16 mode, b2s_sparse_conv_tc_plan_ex with products = 1): one
// fp16 plane per operand, so the gather copies hi rows only, a stage holds [A_hi | W_hi], each K step is one wgmma
// A_hi*W_hi of width N, and the epilogue writes one rounded fp16 plane, or with out_fp32 (b2s_sparse_conv_tc_plan_ex2,
// the training forward and input gradient) fp32 rows as the 3xF16 form does without out_lo.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

using namespace b2s_tc;
// pipeline stages: 4 x (32 KB of gathered rows + 256 N bytes of weights)
constexpr int STAGES = 4;
// GW gather warps with stage ownership: warp w owns every OWN-th K block (pairs of warps share a K block, 64 rows each)
constexpr int GW = 8, OWN = 4;
constexpr int kThreads = 32 * (GW + 8);   // the gather warps, then two consumer warpgroups
constexpr int GROUP = 3;                  // kernel offsets per accumulation chain (Cin = 64)

__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t *bar)
{
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// read-only load the compiler may not move (volatile asm keeps its place among the other volatile asm statements: the
// copies, the barrier operations).  The neighbour-table entries of the NEXT owned K block must be in flight while the
// current one is waited for and copied; as plain __ldg the compiler scheduled them next to their first use, and a third
// of the gather warps' samples were long-scoreboard stalls on them (ncu source counters, round 2).
__device__ __forceinline__ int ld_nc_volatile(const int *ptr)
{
    int v;
    asm volatile("ld.global.nc.s32 %0, [%1];" : "=r"(v) : "l"(ptr));
    return v;
}

struct SpParams {
    const __half *in_hi, *in_lo;
    int in_stride, out_stride;   // halves between consecutive rows of the input / output planes
    int *status;
    const int *nbr;
    const int *n_out_dev;
    const int *perm;             // tile position -> output row (NULL: identity)
    const unsigned *tile_mask;   // per 128-position tile: kernel offsets some row of the tile has (NULL: all)
    int cap_out, K, relu;
    const float *scale, *shift;
    void *out_hi;                // fp16 hi plane, or (out_lo == NULL) fp32 rows [cap_out, COUT]
    __half *out_lo;
    int out_fp32;                // P = 1: fp32 rows in out_hi instead of one fp16 plane
};

// K blocks a tile needs, from its offset mask: bit j = K block j (offsets j*PACK .. j*PACK+PACK-1).  Never empty:
// K block 0 stands in for a tile without any neighbour (cannot happen for SubM / strided conv outputs, but every role
// must agree on the sequence whatever the table holds).
template <int PACK>
__device__ __forceinline__ uint32_t kb_mask_of(uint32_t offsets, int num_kb)
{
    uint32_t m = 0;
    if constexpr (PACK == 1) {
        m = offsets;
    } else {
        constexpr int MAXKB = (27 + PACK - 1) / PACK;
#pragma unroll
        for (int j = 0; j < MAXKB; ++j)
            if (j < num_kb && ((offsets >> (j * PACK)) & ((1u << PACK) - 1u))) m |= 1u << j;
    }
    return m ? m : 1u;
}

// CIN in {8, 16, 32, 64}; COUT in {16, 32, 64}; P in {3, 1}
template <int CIN, int COUT, int P>
__global__ void __launch_bounds__(kThreads, 1)
k_sparse_conv_tc(const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                 const SpParams p)
{
    constexpr int N = COUT;
    constexpr int HALVES = GW / OWN;          // gather warps sharing one K block (each takes BLOCK_M / HALVES rows)
    constexpr int RI = BLOCK_M / HALVES / 4;  // 4-row copy iterations per gather warp and K block
    static_assert(GW % OWN == 0 && RI * 4 * HALVES == BLOCK_M && (OWN & (OWN - 1)) == 0 && RI * STAGES <= 128, "gather warp layout");
    static_assert(CIN <= BLOCK_K && BLOCK_K % CIN == 0, "one K block holds whole kernel offsets");
    constexpr int PACK = BLOCK_K / CIN;                       // kernel offsets per K block
    constexpr int CPO = 8 / PACK;                             // 16-byte chunks per offset inside a 128-byte row
    constexpr int CHAIN_KB = PACK > 1 ? 2 : GROUP;            // K blocks per accumulation chain (short chains)
    constexpr uint32_t CHAIN_BITS = (1u << CHAIN_KB) - 1u;
    constexpr uint32_t B_TILE_BYTES = N * BLOCK_K * ELEM_BYTES;
    static_assert(P == 3 || P == 1, "products per K block: 3 (3xF16) or 1 (f16)");
    constexpr uint32_t STAGE_BYTES = P == 3 ? 2 * A_TILE_BYTES + 2 * B_TILE_BYTES : A_TILE_BYTES + B_TILE_BYTES;
    // B-operand concatenation: the stage holds W_hi (N rows) directly followed by W_lo (N rows), so ONE wgmma with
    // N' = 2N computes A_hi*W_hi (accumulator columns [0,N)) and A_hi*W_lo (columns [N,2N)); a second one (N' = N, the
    // first half of the same accumulator registers) adds A_lo*W_hi into columns [0,N).  8 instead of 12 MMAs per K block
    // for the same products.  The drain adds the two halves.
    constexpr int R = P == 3 ? N : N / 2;                     // accumulator registers per thread: 64 rows x 2N (x N)
    static_assert(N % 16 == 0 && B_TILE_BYTES % 1024 == 0, "wgmma N / swizzle atoms");

    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    __shared__ __align__(8) uint64_t bar_full[STAGES], bar_empty[STAGES];
    __shared__ float s_scale[N], s_shift[N];

    const int warp = warp_idx_uniform(), lane = threadIdx.x & 31;
    const int n_out = min(*p.n_out_dev, p.cap_out);
    const int num_tiles = (n_out + BLOCK_M - 1) / BLOCK_M;
    const int K = p.K;
    const int num_kb = (K + PACK - 1) / PACK;
    const int num_chains = (num_kb + CHAIN_KB - 1) / CHAIN_KB;
    const uint32_t all_offsets = K >= 32 ? 0xffffffffu : ((1u << K) - 1u);
    auto tile_kbm = [&](int tile) -> uint32_t {
        return kb_mask_of<PACK>(p.tile_mask ? __ldg(&p.tile_mask[tile]) & all_offsets : all_offsets, num_kb);
    };

    if (threadIdx.x < N) {
        s_scale[threadIdx.x] = p.scale ? p.scale[threadIdx.x] : 1.f;
        s_shift[threadIdx.x] = p.shift ? p.shift[threadIdx.x] : 0.f;
    }
    if (warp == 1 && lane == 0) {
        for (int i = 0; i < STAGES; ++i) { mbar_init(&bar_full[i], 32 * HALVES + 1); mbar_init(&bar_empty[i], 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < GW) {
        // ===================== gather producers =====================
        // Lane mapping: one warp instruction covers 4 rows x 8 sixteen-byte chunks, so the 32 lanes write 4 whole
        // 128-byte smem rows (bank-conflict free under the 128B swizzle) and read 4 x 128 contiguous global bytes.
        // The loop body is written for instruction count: a gather warp is ONE instruction stream, ~8 cycles per
        // dependent instruction, and the first version of this loop (lambdas, branches around the copies) compiled to
        // ~740 instructions per K block for 32 copies -- the gather warps, not memory, bounded the kernel.
        const int gw = warp;
        const int my_own = gw % OWN;                           // this warp takes K blocks g with g % OWN == my_own
        const int half = gw / OWN;                             // rows half*(128/HALVES) .. of the tile
        const int sub = lane >> 3;                             // row within a group of 4
        const uint32_t chunk = (uint32_t)(lane & 7);           // 16-byte chunk of the 128-byte row
        // row slot rl = half*64 + i*4 + sub (i = 0..RI-1): byte offset rl*128 + ((chunk ^ (rl & 7)) << 4), and
        // rl & 7 = sub for even i, sub + 4 for odd i
        const uint32_t rl0 = (uint32_t)(half * (BLOCK_M / HALVES) + sub);
        const uint32_t sa0 = smem_u32(smem);
        const uint32_t dst_even = rl0 * 128u + ((chunk ^ (uint32_t)sub) << 4);
        const uint32_t dst_odd = rl0 * 128u + ((chunk ^ (uint32_t)(sub + 4)) << 4);
        const int ko = (int)chunk / CPO;                       // offset inside the pack this lane's chunk belongs to
        const char *src_base = reinterpret_cast<const char *>(p.in_hi) + (((int)chunk % CPO) * 16);
        asm volatile("" : "+l"(src_base));                     // one 64-bit register (not base + lane part re-added per copy)
        const long long lo_delta = P == 3 ? reinterpret_cast<const char *>(p.in_lo) - reinterpret_cast<const char *>(p.in_hi) : 0;
        const uint32_t row_bytes = (uint32_t)p.in_stride * ELEM_BYTES;       // rows_in * row_bytes < 2^32 (checked on the host)
        const int grid = (int)gridDim.x;
        const int *__restrict__ nbr = p.nbr;
        const int pos0 = half * (BLOCK_M / HALVES) + sub;      // tile position of row slot i: pos0 + 4 i

        // ---- enumeration of the CTA's K blocks (same sequence in every role); this warp takes every STAGES-th ----
        int e_tile = (int)blockIdx.x - grid;
        uint32_t e_kbm = 0;
        int e_g = 0, e_owned = 0, g_cur = 0;
#define B2S_NEXT_OWNED(KB_OUT, TILE_OUT)                                                      \
        do {                                                                                  \
            KB_OUT = -1;                                                                      \
            for (;;) {                                                                        \
                if (e_kbm == 0) {                                                             \
                    e_tile += grid;                                                           \
                    if (e_tile >= num_tiles) break;                                           \
                    e_kbm = tile_kbm(e_tile);                                                 \
                }                                                                             \
                const int kb_ = __ffs(e_kbm) - 1;                                             \
                e_kbm &= e_kbm - 1;                                                           \
                const bool mine_ = (e_g & (OWN - 1)) == my_own;                               \
                ++e_g;                                                                        \
                if (mine_) { TILE_OUT = e_tile; KB_OUT = kb_; e_owned = e_g - 1; break; }     \
            }                                                                                 \
        } while (0)
        // rows of a tile handled by this lane: index of the row's first table entry (row * K; 0 for a missing row, whose
        // bit in `ok` is clear)
#define B2S_LOAD_ROWS(TILE, RK, OK)                                                           \
        do {                                                                                  \
            OK = 0;                                                                           \
            _Pragma("unroll") for (int i = 0; i < RI; ++i) {                                  \
                const int pos_ = (TILE) * BLOCK_M + pos0 + i * 4;                             \
                const bool live_ = pos_ < n_out;                                              \
                const int row_ = !live_ ? 0 : (p.perm ? __ldg(&p.perm[pos_]) : pos_);         \
                RK[i] = row_ * K;                                                             \
                OK |= (live_ ? 1u : 0u) << i;                                                 \
            }                                                                                 \
        } while (0)
        // table entries of K block KB for the lane's RI rows (k clamped into the table; KV = 0 when k is past the last
        // offset of a partly filled pack)
#define B2S_LOAD_NBR(KB, RK, NB, KV)                                                          \
        do {                                                                                  \
            const int k_ = (KB) * PACK + ko;                                                  \
            KV = k_ < K ? 0xFFFFFFFFu : 0u;                                                   \
            const int *t_ = nbr + (k_ < K ? k_ : K - 1);                                      \
            _Pragma("unroll") for (int i = 0; i < RI; ++i) NB[i] = ld_nc_volatile(t_ + RK[i]); \
        } while (0)

        int rows_cur[RI], rows_pf[RI], nb_cur[RI], nb_nxt[RI];
        uint32_t ok_cur = 0, ok_pf = 0, kv_cur = 0, kv_nxt = 0;
        int cur_tile = -1, nxt_tile = -1, pf_tile = -1;
        int kb_cur;
        B2S_NEXT_OWNED(kb_cur, cur_tile);
        g_cur = e_owned;
        if (kb_cur >= 0) {
            B2S_LOAD_ROWS(cur_tile, rows_cur, ok_cur);
            B2S_LOAD_NBR(kb_cur, rows_cur, nb_cur, kv_cur);
            pf_tile = cur_tile + grid;
            if (pf_tile < num_tiles) B2S_LOAD_ROWS(pf_tile, rows_pf, ok_pf);
        }
        // bit (stage % 4)*RI + i of word stage / 4: this lane's chunk of row slot i in that stage holds zeros
        unsigned long long zeroed_w0 = 0, zeroed_w1 = 0;
        while (kb_cur >= 0) {
            // ---- prefetch the table entries of the next owned K block ----
            int kb_nxt;
            B2S_NEXT_OWNED(kb_nxt, nxt_tile);
            const bool switch_tile = kb_nxt >= 0 && nxt_tile != cur_tile;
            if (kb_nxt >= 0) {
                if (switch_tile) {
                    if (nxt_tile != pf_tile) { B2S_LOAD_ROWS(nxt_tile, rows_pf, ok_pf); pf_tile = nxt_tile; }   // rare: a tile was skipped
                    B2S_LOAD_NBR(kb_nxt, rows_pf, nb_nxt, kv_nxt);
                } else {
                    B2S_LOAD_NBR(kb_nxt, rows_cur, nb_nxt, kv_nxt);
                }
            }
            // ---- current K block: which slots carry a row, which must be written (a row, or zeros over a stale row) ----
            uint32_t valid = 0;
#pragma unroll
            for (int i = 0; i < RI; ++i) valid |= ((uint32_t)(~nb_cur[i]) >> 31) << i;
            valid &= ok_cur & kv_cur;
            const int my_stage = g_cur % STAGES;               // K block g lives in stage g % STAGES, its (g / STAGES)-th use
            const uint32_t use_parity = (((uint32_t)g_cur / STAGES) & 1u) ^ 1u;
            const int zsh = (my_stage & 3) * RI;
            const uint32_t zeroed = (uint32_t)((my_stage < 4 ? zeroed_w0 : zeroed_w1) >> zsh) & ((1u << RI) - 1u);
            const uint32_t need = valid | (~zeroed & ((1u << RI) - 1u));
            const uint32_t sa = sa0 + (uint32_t)my_stage * STAGE_BYTES;
            mbar_wait(&bar_empty[my_stage], use_parity);
            // the K block's weights: its expect_tx arrival is the "+ 1" of the stage's bar_full count
            if (half == 0 && lane == 0) {
                uint8_t *st = smem + (size_t)my_stage * STAGE_BYTES;
                if constexpr (P == 3) {
                    mbar_arrive_expect_tx(&bar_full[my_stage], 2 * B_TILE_BYTES);
                    tma_load_3d(st + 2 * A_TILE_BYTES, &map_w_hi, &bar_full[my_stage], 0, 0, kb_cur);
                    tma_load_3d(st + 2 * A_TILE_BYTES + B_TILE_BYTES, &map_w_lo, &bar_full[my_stage], 0, 0, kb_cur);
                } else {
                    mbar_arrive_expect_tx(&bar_full[my_stage], B_TILE_BYTES);
                    tma_load_3d(st + A_TILE_BYTES, &map_w_hi, &bar_full[my_stage], 0, 0, kb_cur);
                }
            }
            if constexpr (P == 1) {
                // hi rows only
#pragma unroll
                for (int i = 0; i < RI; ++i) {
                    const char *g = src_base + (unsigned long long)(uint32_t)max(nb_cur[i], 0) * row_bytes;
                    asm volatile(
                        "{\n\t.reg .pred p;\n\t"
                        "setp.ne.b32 p, %3, 0;\n\t"
                        "@p cp.async.cg.shared.global [%0], [%1], 16, %2;\n\t}"
                        ::"r"(sa + ((i & 1) ? dst_odd : dst_even) + (uint32_t)i * 512u), "l"(g), "r"((valid >> i & 1u) << 4),
                          "r"(need & (1u << i)) : "memory");
                }
            } else if (lo_delta == (long long)(CIN * ELEM_BYTES)) {
                // interleaved rows [hi Cin | lo Cin]: the lo copy is the hi address + an immediate
#pragma unroll
                for (int i = 0; i < RI; ++i) {
                    const char *g = src_base + (unsigned long long)(uint32_t)max(nb_cur[i], 0) * row_bytes;
                    asm volatile(
                        "{\n\t.reg .pred p;\n\t"
                        "setp.ne.b32 p, %3, 0;\n\t"
                        "@p cp.async.cg.shared.global [%0], [%1], 16, %2;\n\t"
                        "@p cp.async.cg.shared.global [%0+16384], [%1+%4], 16, %2;\n\t}"
                        ::"r"(sa + ((i & 1) ? dst_odd : dst_even) + (uint32_t)i * 512u), "l"(g), "r"((valid >> i & 1u) << 4),
                          "r"(need & (1u << i)), "n"(CIN * ELEM_BYTES) : "memory");
                }
            } else {
#pragma unroll
                for (int i = 0; i < RI; ++i) {
                    const char *g = src_base + (unsigned long long)(uint32_t)max(nb_cur[i], 0) * row_bytes;
                    asm volatile(
                        "{\n\t.reg .pred p;\n\t"
                        "setp.ne.b32 p, %3, 0;\n\t"
                        "@p cp.async.cg.shared.global [%0], [%1], 16, %2;\n\t"
                        "@p cp.async.cg.shared.global [%0+16384], [%4], 16, %2;\n\t}"
                        ::"r"(sa + ((i & 1) ? dst_odd : dst_even) + (uint32_t)i * 512u), "l"(g), "r"((valid >> i & 1u) << 4),
                          "r"(need & (1u << i)), "l"(g + lo_delta) : "memory");
                }
            }
            static_assert(A_TILE_BYTES == 16384, "lo plane of the A tile sits 16384 bytes after the hi plane");
            {
                const unsigned long long clr = ~((unsigned long long)((1u << RI) - 1u) << zsh);
                const unsigned long long set = (unsigned long long)(~valid & ((1u << RI) - 1u)) << zsh;
                if (my_stage < 4) zeroed_w0 = (zeroed_w0 & clr) | set; else zeroed_w1 = (zeroed_w1 & clr) | set;
            }
            cp_async_mbar_arrive_noinc(&bar_full[my_stage]);
            // ---- advance ----
            g_cur = e_owned;
            kb_cur = kb_nxt;
            kv_cur = kv_nxt;
#pragma unroll
            for (int i = 0; i < RI; ++i) nb_cur[i] = nb_nxt[i];
            if (switch_tile) {
#pragma unroll
                for (int i = 0; i < RI; ++i) rows_cur[i] = rows_pf[i];
                ok_cur = ok_pf;
                cur_tile = nxt_tile;
                pf_tile = cur_tile + grid;                  // rows of the tile after this one, long before they are needed
                if (pf_tile < num_tiles) B2S_LOAD_ROWS(pf_tile, rows_pf, ok_pf);
            }
        }
#undef B2S_NEXT_OWNED
#undef B2S_LOAD_ROWS
#undef B2S_LOAD_NBR
        asm volatile("cp.async.wait_all;" ::: "memory");
    } else {
        // ===================== consumers: MMA + epilogue =====================
        const int cg = (warp - GW) >> 2;               // warpgroup: tile rows 64 cg .. 64 cg + 63
        const int wl = warp & 3;
        const uint32_t smem0 = smem_u32(smem);
        const uint32_t a_off = (uint32_t)cg * 64u * 128u;
        int stage = 0;
        uint32_t phase = 0;
        float acc[R], sum[N / 2];
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            uint32_t kbm = tile_kbm(tile);
            // bit set = this K block is the last one of its accumulation chain present in the tile
            uint32_t ce = 0;
            for (int c = 0; c < num_chains; ++c) {
                const uint32_t m_ = kbm & (CHAIN_BITS << (c * CHAIN_KB));
                if (m_) ce |= 0x80000000u >> __clz(m_);
            }
#pragma unroll
            for (int j = 0; j < N / 2; ++j) sum[j] = 0.f;
            uint32_t fresh = 1;                                 // the next MMA opens an accumulation chain
            while (kbm) {
                const uint32_t low = kbm & (0u - kbm);
                kbm ^= low;
                mbar_wait(&bar_full[stage], phase);
                fence_proxy_async();                            // gathered rows were written by cp.async (generic proxy)
                const uint32_t sa = smem0 + (uint32_t)stage * STAGE_BYTES;
                if constexpr (P == 3) {
                    const uint64_t a_hi = make_desc_sw128(sa + a_off), a_lo = make_desc_sw128(sa + A_TILE_BYTES + a_off);
                    const uint64_t b_hl = make_desc_sw128(sa + 2 * A_TILE_BYTES);   // [W_hi; W_lo], 2N rows
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
                        const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                        wgmma_ss<2 * N>(acc, a_hi + koff, b_hl + koff, (fresh && k == 0) ? 0u : 1u);
                        wgmma_ss<N>(acc, a_lo + koff, b_hl + koff, 1);
                    }
                } else {
                    const uint64_t a_hi = make_desc_sw128(sa + a_off), b_hi = make_desc_sw128(sa + A_TILE_BYTES);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
                        const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                        wgmma_ss<N>(acc, a_hi + koff, b_hi + koff, (fresh && k == 0) ? 0u : 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait_all();
                wgmma_fence_operands<R>(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(&bar_empty[stage]);
                __syncwarp();
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
                fresh = (ce & low) ? 1u : 0u;
                if (fresh) {
                    if constexpr (P == 3) {
                        // columns [0,N) hold A_hi*W_hi + A_lo*W_hi, the same columns of the second half A_hi*W_lo
#pragma unroll
                        for (int j = 0; j < R / 2; ++j) sum[j] = __fadd_rn(__fadd_rn(sum[j], acc[j]), acc[R / 2 + j]);
                    } else {
#pragma unroll
                        for (int j = 0; j < R; ++j) sum[j] = __fadd_rn(sum[j], acc[j]);
                    }
                }
            }
            // epilogue: rows m0 = 64 cg + 16 wl + lane/4 and m0 + 8 of the tile, per 8-column block j the channel pair
            // 8j + 2(lane % 4); a quad of lanes writes 16 (fp16 planes) or 32 (fp32) contiguous bytes of a row
            bool range_bad = false;
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int pos = tile * BLOCK_M + cg * 64 + wl * 16 + (lane >> 2) + rh * 8;
                if (pos >= n_out) continue;
                const int row = p.perm ? __ldg(&p.perm[pos]) : pos;
#pragma unroll
                for (int j = 0; j < N / 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    float x0 = fmaf(sum[4 * j + 2 * rh], s_scale[c], s_shift[c]);
                    float x1 = fmaf(sum[4 * j + 2 * rh + 1], s_scale[c + 1], s_shift[c + 1]);
                    if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                    if ((P == 1 && !p.out_fp32) || p.out_lo) {
                        range_bad |= (fabsf(x0) > 65504.f) | (fabsf(x1) > 65504.f);
                        const uint32_t p0 = split_f16(x0), p1 = split_f16(x1);
                        const size_t o = (size_t)row * p.out_stride + c;
                        *reinterpret_cast<uint32_t *>(reinterpret_cast<__half *>(p.out_hi) + o) = __byte_perm(p0, p1, 0x5410);
                        if constexpr (P == 3) *reinterpret_cast<uint32_t *>(p.out_lo + o) = __byte_perm(p0, p1, 0x7632);
                    } else {
                        *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p.out_hi) + (size_t)row * N + c) = make_float2(x0, x1);
                    }
                }
            }
            if (__any_sync(0xffffffffu, range_bad) && lane == 0 && p.status) atomicOr(p.status, B2S_STATUS_F16_RANGE);
        }
    }
}

template <int CIN, int COUT, int P>
int launch(const CUtensorMap &w_hi, const CUtensorMap &w_lo, const SpParams &p, int num_sms, cudaStream_t stream)
{
    constexpr size_t stage = (P == 3 ? 2 : 1) * (A_TILE_BYTES + (size_t)COUT * BLOCK_K * ELEM_BYTES);
    size_t smem = stage * STAGES + 1024;
    B2S_SMEM_OPT_IN((k_sparse_conv_tc<CIN, COUT, P>), smem);
    int tiles_cap = (p.cap_out + BLOCK_M - 1) / BLOCK_M;
    int grid = tiles_cap < num_sms ? tiles_cap : num_sms;
    k_sparse_conv_tc<CIN, COUT, P><<<grid, kThreads, smem, stream>>>(w_hi, w_lo, p);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

extern "C" int b2s_sparse_conv_tc_supported(int cin, int cout)
{
    return (cin == 8 || cin == 16 || cin == 32 || cin == 64) && (cout == 16 || cout == 32 || cout == 64);
}

// Weight layout: Cin = 64: [K][Cout][64]; Cin < 64 (8, 16, 32): packed [ceil(K / (64/Cin))][Cout][64] with column
// (offset-in-pack * Cin + cin) and zero columns for offsets >= K (b2second/tc.py: pack_sparse_weights).
// products = 3: 3xF16 hi/lo planes (out_lo == NULL: fp32 rows).  products = 1: the f16 mode -- feat_lo, w_lo and
// out_lo must be NULL, and the output is one fp16 plane in out_hi, or fp32 rows [cap_out, cout] when out_fp32 is 1
// (out_fp32 must be 0 with products = 3, where out_lo says it).
extern "C" int b2s_sparse_conv_tc_plan_ex2(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in,
                                           int cin, const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K,
                                           const int *num_out_dev, int cap_out, const int *perm,
                                           const unsigned *tile_mask, const float *scale, const float *shift, int relu,
                                           void *out_hi, b2s_half *out_lo, int out_stride, int cout, int products,
                                           int out_fp32, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && feat_lo == nullptr && w_lo == nullptr && out_lo == nullptr),
                "b2s_sparse_conv_tc: products must be 3 (3xF16) or 1 (f16, no lo planes)");
    B2S_REQUIRE(products == 3 ? out_fp32 == 0 : (out_fp32 == 0 || out_fp32 == 1),
                "b2s_sparse_conv_tc: out_fp32 must be 0 or 1 with products = 1 and 0 with products = 3");
    if (products == 1) feat_lo = feat_hi;           // (alignment checks below; the f16 kernel never reads it)
    B2S_REQUIRE(b2s_sparse_conv_tc_supported(cin, cout),
                "b2s_sparse_conv_tc: built for Cin in {8, 16, 32, 64}, Cout in {16, 32, 64} (others: b2s_sparse_conv)");
    B2S_REQUIRE(K >= 1 && K <= 27 && cap_out >= 0 && rows_in >= 0, "b2s_sparse_conv_tc: K must be 1..27");
    B2S_REQUIRE(in_stride >= cin && in_stride % 8 == 0 && ((uintptr_t)feat_hi & 15) == 0 && ((uintptr_t)feat_lo & 15) == 0,
                "b2s_sparse_conv_tc: input rows must be 16-byte aligned (in_stride multiple of 8 halves)");
    B2S_REQUIRE((products == 3 && out_lo == nullptr) || out_fp32 == 1 || (out_stride >= cout && out_stride % 8 == 0 && ((uintptr_t)out_hi & 15) == 0 &&
                                      ((uintptr_t)out_lo & 15) == 0),
                "b2s_sparse_conv_tc: output rows must be 16-byte aligned (out_stride multiple of 8 halves)");
    B2S_REQUIRE((unsigned long long)rows_in * (unsigned long long)in_stride * ELEM_BYTES < (1ull << 32),
                "b2s_sparse_conv_tc: feature planes of 4 GiB or more are not supported (32-bit row offsets)");
    if (cap_out == 0) return 0;
    const int num_sms = num_sms_current();
    CUtensorMap m_hi, m_lo;
    {
        const int pack = BLOCK_K / cin;
        cuuint64_t nkb = (cuuint64_t)((K + pack - 1) / pack);
        cuuint64_t dims[3] = {BLOCK_K, (cuuint64_t)cout, nkb};
        cuuint64_t str[2] = {BLOCK_K * ELEM_BYTES, (cuuint64_t)cout * BLOCK_K * ELEM_BYTES};
        cuuint32_t box[3] = {BLOCK_K, (cuuint32_t)cout, 1};
        if (make_map(&m_hi, w_hi, 3, dims, str, box) || (products == 3 && make_map(&m_lo, w_lo, 3, dims, str, box)))
            return -1;
    }
    SpParams p;
    p.in_hi = reinterpret_cast<const __half *>(feat_hi); p.in_lo = reinterpret_cast<const __half *>(feat_lo);
    p.in_stride = in_stride; p.out_stride = out_stride; p.status = (int *)status_dev;
    p.nbr = nbr; p.n_out_dev = num_out_dev; p.cap_out = cap_out; p.K = K;
    p.perm = perm; p.tile_mask = tile_mask;
    p.relu = relu; p.scale = scale; p.shift = shift; p.out_hi = out_hi; p.out_lo = reinterpret_cast<__half *>(out_lo);
    p.out_fp32 = out_fp32;
#define B2S_TC_CASE(CI, CO)                                                                         \
    if (cin == CI && cout == CO)                                                                    \
        return products == 1 ? launch<CI, CO, 1>(m_hi, m_hi, p, num_sms, stream)                    \
                             : launch<CI, CO, 3>(m_hi, m_lo, p, num_sms, stream);
    B2S_TC_CASE(64, 64) B2S_TC_CASE(64, 32) B2S_TC_CASE(64, 16) B2S_TC_CASE(32, 64) B2S_TC_CASE(32, 32) B2S_TC_CASE(32, 16)
    B2S_TC_CASE(16, 64) B2S_TC_CASE(16, 32) B2S_TC_CASE(16, 16) B2S_TC_CASE(8, 64) B2S_TC_CASE(8, 32) B2S_TC_CASE(8, 16)
#undef B2S_TC_CASE
    b2s_set_error("b2s_sparse_conv_tc: Cin=%d Cout=%d not built", cin, cout);
    return -2;
}

extern "C" int b2s_sparse_conv_tc_plan_ex(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in,
                                          int cin, const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K,
                                          const int *num_out_dev, int cap_out, const int *perm, const unsigned *tile_mask,
                                          const float *scale, const float *shift, int relu, void *out_hi,
                                          b2s_half *out_lo, int out_stride, int cout, int products, unsigned *status_dev,
                                          void *stream)
{
    return b2s_sparse_conv_tc_plan_ex2(feat_hi, feat_lo, in_stride, rows_in, cin, w_hi, w_lo, nbr, K, num_out_dev,
                                       cap_out, perm, tile_mask, scale, shift, relu, out_hi, out_lo, out_stride, cout,
                                       products, 0, status_dev, stream);
}

// the 3xF16 form
extern "C" int b2s_sparse_conv_tc_plan(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                                       const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K,
                                       const int *num_out_dev, int cap_out, const int *perm, const unsigned *tile_mask,
                                       const float *scale, const float *shift, int relu, void *out_hi, b2s_half *out_lo,
                                       int out_stride, int cout, unsigned *status_dev, void *stream)
{
    return b2s_sparse_conv_tc_plan_ex(feat_hi, feat_lo, in_stride, rows_in, cin, w_hi, w_lo, nbr, K, num_out_dev, cap_out,
                                      perm, tile_mask, scale, shift, relu, out_hi, out_lo, out_stride, cout, 3, status_dev,
                                      stream);
}

extern "C" int b2s_sparse_conv_tc(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in, int cin,
                                  const b2s_half *w_hi, const b2s_half *w_lo, const int *nbr, int K,
                                  const int *num_out_dev, int cap_out, const float *scale, const float *shift, int relu,
                                  void *out_hi, b2s_half *out_lo, int out_stride, int cout, unsigned *status_dev,
                                  void *stream_)
{
    return b2s_sparse_conv_tc_plan(feat_hi, feat_lo, in_stride, rows_in, cin, w_hi, w_lo, nbr, K, num_out_dev, cap_out,
                                   nullptr, nullptr, scale, shift, relu, out_hi, out_lo, out_stride, cout, status_dev,
                                   stream_);
}
