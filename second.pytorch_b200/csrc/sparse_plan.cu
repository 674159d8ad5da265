// sparse_plan.cu -- tile plan of a sparse convolution (b2s_sparse_tile_plan): which kernel offsets a 128-row output
// tile needs at all, and an order of the output rows that makes that set small.
//
// b2s_sparse_conv_tc is output-stationary: a CTA owns 128 output rows (one accumulator tile) and multiplies, per
// kernel offset k, the 128 gathered neighbour rows with W[k].  Only ~3.5-9 of the 27 neighbours of a row exist
// (SURVEY.md App. D), so most gathered rows are zeros -- but an offset can only be SKIPPED when none of the tile's 128
// rows has that neighbour.  In storage order that removes ~25 % of the (tile, offset) blocks (measured on the bench
// clouds); when rows with a similar neighbourhood shape share a tile it is ~45 %:
//   class(row) = [some neighbour in the planes below the centre] [.. above] [in the centre plane: rows before the
//                centre row] [.. after]                                        (4 bits; 2 bits for a k x 1 x 1 kernel)
// Rows are grouped by class inside chunks of 8192 consecutive rows (stable, so a tile's rows stay spatial neighbours
// and the gather stays L2-friendly; one CTA per chunk, no global scan):  perm[pos] = row,  tiles = 128 consecutive
// positions,  tile_mask[tile] = OR of the rows' offset masks.
// The conv kernel's result does not depend on the order or the masks (a missing neighbour contributes exact zeros and
// its accumulation chains have fixed offset boundaries), so planned and unplanned runs are bit-identical.
#include "common.cuh"

namespace {

constexpr int kChunkRows = 8192;          // rows per CTA (64 tiles)
constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kRowsPerWarp = kChunkRows / kWarps;     // 256
constexpr int kClasses = 16;

struct PlanGeom {
    int K;
    unsigned below, above, before, after;   // offset masks of the four class groups
    unsigned all;                           // (1 << K) - 1
};

// offset mask of the 32 rows row0 .. row0+31 (lane = row): K coalesced 32-int loads + ballots, then a funnel shift
__device__ __forceinline__ unsigned warp_row_masks(const int *__restrict__ nbr, long long row0, int n_rows, int K,
                                                   unsigned *s_bits /* >= 28 words of this warp */)
{
    const int lane = threadIdx.x & 31;
    const long long base = row0 * K;
    const long long end = (long long)n_rows * K;
    // all K (<= 27) loads first, then the ballots: one L2 round trip per 32 rows instead of K
    int v[27];
#pragma unroll
    for (int j = 0; j < 27; ++j) {
        const long long f = base + (long long)j * 32 + lane;
        v[j] = (j < K && f < end) ? __ldg(&nbr[f]) : -1;
    }
#pragma unroll
    for (int j = 0; j < 27; ++j) {
        const unsigned b = __ballot_sync(0xffffffffu, v[j] >= 0);
        if (lane == 0 && j < K) s_bits[j] = b;
    }
    if (lane == 0) s_bits[K] = 0u;
    __syncwarp();
    const int bit0 = lane * K;                       // first bit of this lane's row in the K*32-bit array
    const unsigned lo = s_bits[bit0 >> 5], hi = s_bits[(bit0 >> 5) + 1];
    const unsigned m = __funnelshift_r(lo, hi, bit0 & 31) & (K >= 32 ? 0xffffffffu : ((1u << K) - 1u));
    __syncwarp();
    return m;
}

__device__ __forceinline__ int row_class(unsigned m, const PlanGeom &g)
{
    return ((m & g.below) ? 1 : 0) | ((m & g.above) ? 2 : 0) | ((m & g.before) ? 4 : 0) | ((m & g.after) ? 8 : 0);
}

// One CTA per chunk of kChunkRows rows.
//   sort == 0: tile_mask only (rows stay in storage order, perm untouched / may be NULL)
//   sort == 1: stable grouping by class inside the chunk -> perm, tile_mask over the grouped order
__global__ void __launch_bounds__(kThreads, 1)
k_tile_plan(const int *__restrict__ nbr, const unsigned *__restrict__ row_mask, const int *__restrict__ n_dev, int cap,
            PlanGeom g, int sort, int *perm, unsigned *tile_mask)
{
    extern __shared__ unsigned s_dyn[];
    unsigned *s_mask = s_dyn;                                        // [kChunkRows] offset mask per row
    unsigned short *s_order = reinterpret_cast<unsigned short *>(s_dyn + kChunkRows);   // [kChunkRows] grouped -> local row
    __shared__ int s_cnt[kClasses][kWarps + 1];                      // per class and warp: rows (then exclusive base)
    __shared__ unsigned s_bits[kWarps][32];
    const int n = min(*n_dev, cap);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (long long chunk0 = (long long)blockIdx.x * kChunkRows; chunk0 < n; chunk0 += (long long)gridDim.x * kChunkRows) {
        const int rows_here = (int)min((long long)kChunkRows, (long long)n - chunk0);
        // ---- pass 1: row masks (+ per-warp class counts) ----
        if (sort) {                                                  // s_cnt[c][w]: rows of class c in warp w's span
            for (int i = threadIdx.x; i < kClasses * (kWarps + 1); i += kThreads) (&s_cnt[0][0])[i] = 0;
            __syncthreads();
        }
        unsigned pre[kRowsPerWarp / 32];                             // masks handed over by the rulebook builder: one load each
        if (row_mask) {
#pragma unroll
            for (int q = 0; q < kRowsPerWarp / 32; ++q) {
                const int i = warp * kRowsPerWarp + q * 32 + lane;
                pre[q] = i < rows_here ? __ldg(&row_mask[chunk0 + i]) & g.all : 0u;
            }
        }
#pragma unroll
        for (int s = 0; s < kRowsPerWarp; s += 32) {
            const int local = warp * kRowsPerWarp + s;
            unsigned m = 0;
            if (row_mask) m = pre[s / 32];
            else if (local < rows_here) m = warp_row_masks(nbr, chunk0 + local, n, g.K, s_bits[warp]);
            const bool live = local + lane < rows_here;
            if (!live) m = 0;
            s_mask[local + lane] = m;
            if (sort) {
                // one match instead of 16 ballots: lanes of the same class find each other, the lowest one counts them
                const int c = live ? row_class(m, g) : kClasses + lane;
                const unsigned peers = __match_any_sync(0xffffffffu, c);
                if (live && (peers & ((1u << lane) - 1u)) == 0u) s_cnt[c][warp] += __popc(peers);
                __syncwarp();
            }
        }
        if (sort) {
            __syncthreads();
            // exclusive scan over (class major, warp minor): 16 x 32 entries, one warp
            if (warp == 0) {
                int carry = 0;
                for (int c = 0; c < kClasses; ++c) {
                    const int v = s_cnt[c][lane];
                    int inc = v;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int t = __shfl_up_sync(0xffffffffu, inc, o);
                        if (lane >= o) inc += t;
                    }
                    s_cnt[c][lane] = carry + inc - v;
                    carry += __shfl_sync(0xffffffffu, inc, 31);
                }
            }
            __syncthreads();
            // ---- pass 2: stable scatter of the local row numbers ----
            // s_cnt[c][warp] is now this warp's next free position of class c (only this warp touches its column)
            for (int s = 0; s < kRowsPerWarp; s += 32) {
                const int local = warp * kRowsPerWarp + s + lane;
                const bool live = local < rows_here;
                const int c = live ? row_class(s_mask[local], g) : kClasses + lane;
                const unsigned peers = __match_any_sync(0xffffffffu, c);
                const int leader = __ffs(peers) - 1;
                int base = 0;
                if (live && lane == leader) { base = s_cnt[c][warp]; s_cnt[c][warp] = base + __popc(peers); }
                base = __shfl_sync(0xffffffffu, base, leader);
                if (live) s_order[base + __popc(peers & ((1u << lane) - 1u))] = (unsigned short)local;
                __syncwarp();
            }
            __syncthreads();
            for (int i = threadIdx.x; i < rows_here; i += kThreads) perm[chunk0 + i] = (int)(chunk0 + s_order[i]);
        } else {
            __syncthreads();
        }
        // ---- tile masks: OR over the 128 rows of each tile (a warp per tile, 4 rows per lane) ----
        const int tiles_here = (rows_here + 127) / 128;
        for (int t = warp; t < tiles_here; t += kWarps) {
            unsigned m = 0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int i = t * 128 + q * 32 + lane;
                if (i < rows_here) m |= s_mask[sort ? s_order[i] : i];
            }
            m = __reduce_or_sync(0xffffffffu, m);
            if (lane == 0) tile_mask[chunk0 / 128 + t] = m;
        }
        __syncthreads();
    }
}

}  // namespace

extern "C" int b2s_sparse_tile_plan(const int *nbr, const unsigned *row_mask, int K, const int *ksize, const int *num_out_dev,
                                    int cap_out, int sort, int *perm, unsigned *tile_mask, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(K >= 1 && K <= 27 && cap_out >= 0, "b2s_sparse_tile_plan: K must be 1..27");
    B2S_REQUIRE(tile_mask != nullptr && (sort == 0 || perm != nullptr), "b2s_sparse_tile_plan: tile_mask (and perm when sort=1) required");
    if (cap_out == 0) return 0;
    PlanGeom g;
    g.K = K;
    g.below = g.above = g.before = g.after = 0u;
    g.all = K >= 32 ? 0xffffffffu : ((1u << K) - 1u);
    int kz = K, ky = 1, kx = 1;
    if (ksize) { kz = ksize[0]; ky = ksize[1]; kx = ksize[2]; }
    B2S_REQUIRE(kz >= 1 && ky >= 1 && kx >= 1 && kz * ky * kx == K, "b2s_sparse_tile_plan: ksize does not multiply to K");
    for (int k = 0; k < K; ++k) {
        const int z = k / (ky * kx), y = (k / kx) % ky;
        if (2 * z + 1 < kz) g.below |= 1u << k;
        else if (2 * z + 1 > kz) g.above |= 1u << k;
        else if (2 * y + 1 < ky) g.before |= 1u << k;
        else if (2 * y + 1 > ky) g.after |= 1u << k;
    }
    const size_t smem = sizeof(unsigned) * kChunkRows + sizeof(unsigned short) * kChunkRows;
    static bool attr_done[64] = {false};
    int dev = 0;
    B2S_CUDA_OK(cudaGetDevice(&dev));
    if (!attr_done[dev & 63]) {
        B2S_CUDA_OK(cudaFuncSetAttribute(k_tile_plan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[dev & 63] = true;
    }
    int grid = b2s_cdiv(cap_out, kChunkRows);
    if (grid > 132 * 2) grid = 132 * 2;
    B2S_REQUIRE(nbr != nullptr || row_mask != nullptr, "b2s_sparse_tile_plan: nbr or row_mask required");
    k_tile_plan<<<grid, kThreads, smem, stream>>>(nbr, row_mask, num_out_dev, cap_out, g, sort ? 1 : 0, perm, tile_mask);
    B2S_LAUNCH_OK();
    return 0;
}
