// sparse_grad.cu -- backward of the sparse convolution and of dense() (include/b2second.h, "sparse convolution
// backward"): the weight gradient (b2s_sparse_conv_wgrad), the input-side neighbour table of a strided conv
// (b2s_rulebook_transpose), the gather from a BEV gradient back into rows (b2s_from_bev) and the automatically scaled
// 3xF16 split of a gradient (b2s_split_f16_autoscale) and the packed, scaled weight planes of a layer in training
// (b2s_pack_sparse_weights), and with the same scale rule the weight planes of a dense 3x3 RPN layer in training
// (b2s_pack_conv2d_weights, used with conv_train.cu).  The input gradient itself is the forward kernels on a
// transposed table (sparse_conv.cu, sparse_conv_tc.cu).
//
// Weight gradient in fp32 (b2s_sparse_conv_wgrad; the tensor-pipe version is further down): dW[k][ci][co] =
// sum_o X[nbr[o][k]][ci] * dY[o][co], a reduction over ROWS.  Launch 1: one CTA per
// (2048-row slab of output rows, kernel offset k, 64x64 tile of (ci, co)); 256 threads as 16 x 16, thread (ty, tx)
// owns ci = ty + 16a, co = tx + 16b (a < A, b < B) of the tile, in fp32 registers.  Per 32-row chunk the gathered X rows
// (zeros for a missing neighbour) and the dY rows go to shared memory; rows are added in ascending order.  The slab's
// partial goes to the workspace; launch 2 adds the slabs in ascending order.  No float atomics: the result depends only
// on the table and the values, never on scheduling.
#include <cuda_fp16.h>

#include "autoscale.cuh"
#include "tc_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int WG_SLAB = 2048;   // output rows per partial sum
constexpr int WG_CHUNK = 32;    // rows staged in shared memory at a time
constexpr int WG_TILE = 64;     // (ci, co) tile of one CTA
constexpr int WG_LD = WG_TILE + 1;

inline int grid_for(long long items)
{
    long long b = (items + kThreads - 1) / kThreads;
    return (int)(b < 1 ? 1 : (b < 132 * 8 ? b : 132 * 8));
}

inline int num_slabs(int cap_out) { return (cap_out + WG_SLAB - 1) / WG_SLAB; }

template <int A, int B>
__global__ void __launch_bounds__(kThreads)
k_wgrad_partial(const float *__restrict__ x, int cin, const float *__restrict__ dy, int cout,
                const int *__restrict__ nbr, int K, const int *__restrict__ n_out_dev, int cap_out,
                float *__restrict__ partial)
{
    __shared__ float s_x[WG_CHUNK][WG_LD];
    __shared__ float s_y[WG_CHUNK][WG_LD];
    __shared__ int s_src[WG_CHUNK];
    const int n_out = min(*n_out_dev, cap_out);
    const int slab = blockIdx.x, k = blockIdx.y;
    const int row0 = slab * WG_SLAB;
    if (row0 >= n_out) return;                      // launch 2 reads only the slabs below n_out
    const int tiles_co = (cout + WG_TILE - 1) / WG_TILE;
    const int ci0 = (int)(blockIdx.z / tiles_co) * WG_TILE, co0 = (int)(blockIdx.z % tiles_co) * WG_TILE;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int row_end = min(row0 + WG_SLAB, n_out);

    float acc[A][B];
#pragma unroll
    for (int a = 0; a < A; ++a)
#pragma unroll
        for (int b = 0; b < B; ++b) acc[a][b] = 0.f;

    for (int c0 = row0; c0 < row_end; c0 += WG_CHUNK) {
        const int rows = min(WG_CHUNK, row_end - c0);
        int have = 0;
        if (tid < WG_CHUNK) {
            const int src = tid < rows ? __ldg(&nbr[(size_t)(c0 + tid) * K + k]) : -1;
            s_src[tid] = src;
            have = src >= 0;
        }
        if (!__syncthreads_or(have)) continue;      // block-uniform: no row of the chunk has this neighbour
        for (int i = tid; i < WG_CHUNK * WG_TILE; i += kThreads) {
            const int r = i / WG_TILE, c = i - r * WG_TILE;
            const int src = s_src[r];
            const int ci = ci0 + c, co = co0 + c;
            s_x[r][c] = (src >= 0 && ci < cin) ? __ldg(&x[(size_t)src * cin + ci]) : 0.f;
            s_y[r][c] = (src >= 0 && co < cout) ? __ldg(&dy[(size_t)(c0 + r) * cout + co]) : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int r = 0; r < WG_CHUNK; ++r) {
            float xv[A], yv[B];
#pragma unroll
            for (int a = 0; a < A; ++a) xv[a] = s_x[r][ty + 16 * a];
#pragma unroll
            for (int b = 0; b < B; ++b) yv[b] = s_y[r][tx + 16 * b];
#pragma unroll
            for (int a = 0; a < A; ++a)
#pragma unroll
                for (int b = 0; b < B; ++b) acc[a][b] = fmaf(xv[a], yv[b], acc[a][b]);
        }
        __syncthreads();
    }
    float *dst = partial + ((size_t)slab * K + k) * cin * cout;
#pragma unroll
    for (int a = 0; a < A; ++a) {
        const int ci = ci0 + ty + 16 * a;
        if (ci >= cin) continue;
#pragma unroll
        for (int b = 0; b < B; ++b) {
            const int co = co0 + tx + 16 * b;
            if (co < cout) dst[(size_t)ci * cout + co] = acc[a][b];
        }
    }
}

__global__ void k_wgrad_reduce(const float *__restrict__ partial, long long elems, const int *__restrict__ n_out_dev,
                               int cap_out, const float *__restrict__ scale_dev, float *__restrict__ dw)
{
    const int n_out = min(*n_out_dev, cap_out);
    const int slabs = (n_out + WG_SLAB - 1) / WG_SLAB;
    const float sc = scale_dev ? __ldg(scale_dev) : 1.f;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < elems;
         e += (long long)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int j = 0; j < slabs; ++j) s += __ldg(&partial[(size_t)j * elems + e]);
        dw[e] = scale_dev ? s * sc : s;
    }
}

template <int A, int B>
void launch_partial(const float *x, int cin, const float *dy, int cout, const int *nbr, int K, const int *n_out_dev,
                    int cap_out, float *partial, cudaStream_t stream)
{
    const int tiles = ((cin + WG_TILE - 1) / WG_TILE) * ((cout + WG_TILE - 1) / WG_TILE);
    k_wgrad_partial<A, B><<<dim3(num_slabs(cap_out), K, tiles), kThreads, 0, stream>>>(x, cin, dy, cout, nbr, K,
                                                                                       n_out_dev, cap_out, partial);
}

__global__ void k_rulebook_transpose(const int *__restrict__ nbr, const int *__restrict__ n_out_dev, int cap_out, int K,
                                     int *__restrict__ nbrT, int cap_in, unsigned *__restrict__ status)
{
    const long long total = (long long)min(*n_out_dev, cap_out) * K;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const int i = __ldg(&nbr[e]);
        if (i < 0) continue;
        const int o = (int)(e / K), k = (int)(e - (long long)o * K);
        if (i >= cap_in) {
            if (status) atomicOr(status, B2S_STATUS_ROWS_OVERFLOW);
            continue;
        }
        nbrT[(size_t)i * K + k] = o;
    }
}

__global__ void k_from_bev(const float *__restrict__ dmap, const int *__restrict__ coors, const int *__restrict__ n_dev,
                           int cap_rows, int C, int batch, int D, int H, int W, int layout, float *__restrict__ drows)
{
    const int n = min(*n_dev, cap_rows);
    const long long total = (long long)n * C;
    for (long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x; gid < total;
         gid += (long long)gridDim.x * blockDim.x) {
        const int row = (int)(gid / C), c = (int)(gid % C);
        const int4 q = __ldg(reinterpret_cast<const int4 *>(coors + (size_t)row * 4));  // b,z,y,x
        float v = 0.f;
        if ((unsigned)q.x < (unsigned)batch && (unsigned)q.y < (unsigned)D && (unsigned)q.z < (unsigned)H &&
            (unsigned)q.w < (unsigned)W) {
            const size_t CD = (size_t)C * D;
            const size_t ch = (size_t)c * D + q.y;
            const size_t idx = layout == B2S_LAYOUT_NCHW ? (((size_t)q.x * CD + ch) * H + q.z) * W + q.w
                                                         : (((size_t)q.x * H + q.z) * W + q.w) * CD + ch;
            v = __ldg(&dmap[idx]);
        }
        drows[gid] = v;
    }
}

// one thread per 8 columns of a packed row: out[kb, o, p * n_in' + i] = L[kb * P + p, i, o] * s, zero past K and n_in
// (tc.pack_sparse_weights), split into hi / lo (P = 1: hi only).  s is the float32 the host path multiplies by:
// float(2.0 ** e).
template <int P>
__global__ void k_pack_sparse_weights(const float *__restrict__ w, int K, int cin, int cout, int transpose, int flip,
                                      int n_in, int n_in_pad, int n_out, int nkb, __half *__restrict__ hi,
                                      __half *__restrict__ lo, float *__restrict__ scale_dev)
{
    const int e = autoscale_exponent(*reinterpret_cast<const volatile unsigned *>(scale_dev + 2));
    const float s = (float)ldexp(1.0, e);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        scale_dev[0] = s;
        scale_dev[1] = (float)ldexp(1.0, -e);
    }
    const int pack = b2s_tc::BLOCK_K / n_in_pad;
    const long long n = (long long)nkb * n_out * (b2s_tc::BLOCK_K / 8);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / (b2s_tc::BLOCK_K / 8);            // (kb, o)
        const int c0 = (int)(i - row * (b2s_tc::BLOCK_K / 8)) * 8;
        const int kb = (int)(row / n_out), o = (int)(row - (long long)kb * n_out);
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int col = c0 + j, p = col / n_in_pad, ci = col - p * n_in_pad, k = kb * pack + p;
            float x = 0.f;
            if (k < K && ci < n_in) {
                const int ks = flip ? K - 1 - k : k;
                x = transpose ? __ldg(&w[((size_t)ks * cin + o) * cout + ci]) : __ldg(&w[((size_t)ks * cin + ci) * cout + o]);
            }
            v[j] = __fmul_rn(x, s);
        }
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t pa = b2s_tc::split_f16_keep_nonfinite(v[2 * j]),
                           pb = b2s_tc::split_f16_keep_nonfinite(v[2 * j + 1]);
            h[j] = __byte_perm(pa, pb, 0x5410);
            l[j] = __byte_perm(pa, pb, 0x7632);
        }
        *reinterpret_cast<uint4 *>(hi + row * b2s_tc::BLOCK_K + c0) = make_uint4(h[0], h[1], h[2], h[3]);
        if constexpr (P == 3)
            *reinterpret_cast<uint4 *>(lo + row * b2s_tc::BLOCK_K + c0) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

// dense 3x3 weights, one thread per 8 columns of a packed row: out[g, tap, o, i] = L[tap][g * 128 + o][i] * s with
// L[tap][o][i] = W[o][i][tap] (transpose 0: the forward) or W[i][o][8 - tap] (transpose 1: the input gradient), W the
// torch weight [cout, cin, 3, 3]; rows past n_out of the last group are zero.  s as in k_pack_sparse_weights.
template <int P>
__global__ void k_pack_conv2d_weights(const float *__restrict__ w, int cout, int cin, int transpose, int n_in,
                                      int n_out, int n_pad, int groups, __half *__restrict__ hi, __half *__restrict__ lo,
                                      float *__restrict__ scale_dev)
{
    const int e = autoscale_exponent(*reinterpret_cast<const volatile unsigned *>(scale_dev + 2));
    const float s = (float)ldexp(1.0, e);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        scale_dev[0] = s;
        scale_dev[1] = (float)ldexp(1.0, -e);
    }
    const int cols = n_in / 8;
    const long long n = (long long)groups * 9 * n_pad * cols;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / cols;                               // (g, tap, o)
        const int c0 = (int)(i - row * cols) * 8;
        const int o = (int)(row % n_pad), tap = (int)((row / n_pad) % 9), g = (int)(row / ((long long)n_pad * 9));
        const int oo = g * 128 + o;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int ii = c0 + j;
            float x = 0.f;
            if (oo < n_out)
                x = transpose ? __ldg(&w[((size_t)ii * cin + oo) * 9 + (8 - tap)]) : __ldg(&w[((size_t)oo * cin + ii) * 9 + tap]);
            v[j] = __fmul_rn(x, s);
        }
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t pa = b2s_tc::split_f16_keep_nonfinite(v[2 * j]),
                           pb = b2s_tc::split_f16_keep_nonfinite(v[2 * j + 1]);
            h[j] = __byte_perm(pa, pb, 0x5410);
            l[j] = __byte_perm(pa, pb, 0x7632);
        }
        *reinterpret_cast<uint4 *>(hi + row * n_in + c0) = make_uint4(h[0], h[1], h[2], h[3]);
        if constexpr (P == 3) *reinterpret_cast<uint4 *>(lo + row * n_in + c0) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

template <int P>
__global__ void k_split_f16_scaled(const float *__restrict__ x, __half *__restrict__ hi, __half *__restrict__ lo,
                                   const int *__restrict__ n_rows_dev, int cap_rows, int row_floats, int out_channels,
                                   int out_stride, float *__restrict__ scale_dev)
{
    const int e = autoscale_exponent(*reinterpret_cast<const volatile unsigned *>(scale_dev + 1));
    const float s = ldexpf(1.f, e);
    if (blockIdx.x == 0 && threadIdx.x == 0) scale_dev[0] = ldexpf(1.f, -e);
    const int groups = out_channels / 8;
    const long long n = (long long)(n_rows_dev ? min(*n_rows_dev, cap_rows) : cap_rows) * groups;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / groups;
        const int c0 = (int)(i - row * groups) * 8;
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = c0 + 2 * j;
            const float a = c < row_floats ? __ldg(&x[row * row_floats + c]) * s : 0.f;    // power of two: exact
            const float b = c + 1 < row_floats ? __ldg(&x[row * row_floats + c + 1]) * s : 0.f;
            const uint32_t pa = b2s_tc::split_f16_keep_nonfinite(a), pb = b2s_tc::split_f16_keep_nonfinite(b);
            h[j] = __byte_perm(pa, pb, 0x5410);
            l[j] = __byte_perm(pa, pb, 0x7632);
        }
        *reinterpret_cast<uint4 *>(hi + row * out_stride + c0) = make_uint4(h[0], h[1], h[2], h[3]);
        if constexpr (P == 3) *reinterpret_cast<uint4 *>(lo + row * out_stride + c0) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}


// ---- weight gradient on the tensor pipe (b2s_sparse_conv_wgrad_tc) ---------------------------------------------------
// D[64, Cout] = sum over rows of A[64, rows] * B[Cout, rows]^T with A = X^T of one K block (PACK = 64/Cin kernel offsets
// side by side, m = offset_in_pack * Cin + ci, the forward's packing) and B = dY^T.  One warpgroup per CTA owns one
// (2048-position slab, K block).  Per 64-position chunk (positions in `perm` order, one half of a 128-position tile) the
// gathered X rows and the dY rows are transposed while they are staged, into the SAME K-major SWIZZLE_128B layout the
// forward's operands use (element (m, r) at m*128 + (((r/8) ^ (m%8)) << 4) + (r%8)*2): 16-byte global loads, 2-byte
// shared stores.  Four k16 steps per chunk issue A_hi*[B_hi; B_lo] (N' = 2 Cout) + A_lo*B_hi; each chunk is one
// accumulation chain, drained into fp32 running sums with round-to-nearest adds.  A chunk whose rows have no neighbour
// in the K block -- known from tile_mask, or found while staging -- contributes exact zeros and is skipped, so results are
// bit-identical with and without tile_mask.  The slab partials go to the workspace; the reduce launch adds them in
// order, multiplies by *scale_dev and unpacks into [K, Cin, Cout].
//
// P = products per k16 step: 3 (3xF16, above) or 1 (the f16 mode, b2s_sparse_conv_wgrad_tc_ex with products = 1): one
// fp16 plane per operand, so staging moves the hi rows only (half the bytes), the smem holds [A_hi | B_hi], each k16
// step is one wgmma A_hi*B_hi of width N, and the chain's accumulator (64 x N) is drained as it is.  The partials have
// the same layout, so the workspace is the same.
constexpr int WT_CHUNK = 64;
constexpr int WT_THREADS = 128;

__device__ __forceinline__ uint32_t sw128_off(int m, int r)
{
    return (uint32_t)(m * 128 + ((((r >> 3) ^ (m & 7)) << 4) | ((r & 7) << 1)));
}

template <int CIN, int COUT, int P>
__global__ void __launch_bounds__(WT_THREADS)
k_wgrad_tc(const __half *__restrict__ x_hi, const __half *__restrict__ x_lo, int in_stride,
           const __half *__restrict__ g_hi, const __half *__restrict__ g_lo, int g_stride, const int *__restrict__ nbr,
           int K, const int *__restrict__ n_out_dev, int cap_out, const int *__restrict__ perm,
           const unsigned *__restrict__ tile_mask, float *__restrict__ partial)
{
    using namespace b2s_tc;
    constexpr int N = COUT;
    constexpr int PACK = b2s_tc::BLOCK_K / CIN;
    constexpr int A_BYTES = 64 * 128;
    static_assert(P == 3 || P == 1, "products per k16 step: 3 (3xF16) or 1 (f16)");
    constexpr int R = P == 3 ? N : N / 2;                    // accumulator registers: 64 rows x 2N (x N) columns
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    // P = 3: sb = [B_hi (N rows); B_lo (N rows)]; P = 1: [A_hi | B_hi]
    uint8_t *sa_hi = smem, *sa_lo = smem + A_BYTES, *sb = smem + (P == 3 ? 2 : 1) * A_BYTES;
    __shared__ int s_row[WT_CHUNK];

    const int n_out = min(*n_out_dev, cap_out);
    const int slab = blockIdx.x, kb = blockIdx.y, num_kb = gridDim.y;
    const int pos0 = slab * WG_SLAB;
    if (pos0 >= n_out) return;
    const int pos_end = min(pos0 + WG_SLAB, n_out);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t all_offsets = K >= 32 ? 0xffffffffu : ((1u << K) - 1u);
    const uint32_t pack_bits = (((1u << PACK) - 1u) << (kb * PACK)) & all_offsets;

    float acc[R], sum[N / 2];
#pragma unroll
    for (int j = 0; j < N / 2; ++j) sum[j] = 0.f;

    for (int c0 = pos0; c0 < pos_end; c0 += WT_CHUNK) {
        if (tile_mask && !(__ldg(&tile_mask[c0 / BLOCK_M]) & pack_bits)) continue;   // uniform: no row needs the block
        if (tid < WT_CHUNK) {
            const int pos = c0 + tid;
            s_row[tid] = pos < pos_end ? (perm ? __ldg(&perm[pos]) : pos) : -1;
        }
        __syncthreads();
        int have = 0;
        // A = X^T: (row r, 8 consecutive m) per item; m0 / CIN = offset in the pack, m0 % CIN = first channel
        for (int v = tid; v < WT_CHUNK * 8; v += WT_THREADS) {
            const int r = v >> 3, m0 = (v & 7) * 8;
            const int k = kb * PACK + m0 / CIN, ci0 = m0 % CIN;
            const int row = s_row[r];
            const int src = (row >= 0 && k < K) ? __ldg(&nbr[(size_t)row * K + k]) : -1;
            if constexpr (P == 3) {
                uint4 h = make_uint4(0, 0, 0, 0), l = make_uint4(0, 0, 0, 0);
                if (src >= 0) {
                    h = __ldg(reinterpret_cast<const uint4 *>(x_hi + (size_t)src * in_stride + ci0));
                    l = __ldg(reinterpret_cast<const uint4 *>(x_lo + (size_t)src * in_stride + ci0));
                    have = 1;
                }
                const uint16_t *hh = reinterpret_cast<const uint16_t *>(&h), *ll = reinterpret_cast<const uint16_t *>(&l);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    *reinterpret_cast<uint16_t *>(sa_hi + sw128_off(m0 + j, r)) = hh[j];
                    *reinterpret_cast<uint16_t *>(sa_lo + sw128_off(m0 + j, r)) = ll[j];
                }
            } else {
                uint4 h = make_uint4(0, 0, 0, 0);
                if (src >= 0) {
                    h = __ldg(reinterpret_cast<const uint4 *>(x_hi + (size_t)src * in_stride + ci0));
                    have = 1;
                }
                const uint16_t *hh = reinterpret_cast<const uint16_t *>(&h);
#pragma unroll
                for (int j = 0; j < 8; ++j) *reinterpret_cast<uint16_t *>(sa_hi + sw128_off(m0 + j, r)) = hh[j];
            }
        }
        // B = dY^T: (row r, 8 consecutive output channels) per item
        for (int v = tid; v < WT_CHUNK * (N / 8); v += WT_THREADS) {
            const int r = v / (N / 8), n0 = (v % (N / 8)) * 8;
            const int row = s_row[r];
            if constexpr (P == 3) {
                uint4 h = make_uint4(0, 0, 0, 0), l = make_uint4(0, 0, 0, 0);
                if (row >= 0) {
                    h = __ldg(reinterpret_cast<const uint4 *>(g_hi + (size_t)row * g_stride + n0));
                    l = __ldg(reinterpret_cast<const uint4 *>(g_lo + (size_t)row * g_stride + n0));
                }
                const uint16_t *hh = reinterpret_cast<const uint16_t *>(&h), *ll = reinterpret_cast<const uint16_t *>(&l);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    *reinterpret_cast<uint16_t *>(sb + sw128_off(n0 + j, r)) = hh[j];
                    *reinterpret_cast<uint16_t *>(sb + sw128_off(N + n0 + j, r)) = ll[j];
                }
            } else {
                uint4 h = make_uint4(0, 0, 0, 0);
                if (row >= 0) h = __ldg(reinterpret_cast<const uint4 *>(g_hi + (size_t)row * g_stride + n0));
                const uint16_t *hh = reinterpret_cast<const uint16_t *>(&h);
#pragma unroll
                for (int j = 0; j < 8; ++j) *reinterpret_cast<uint16_t *>(sb + sw128_off(n0 + j, r)) = hh[j];
            }
        }
        fence_proxy_async();                                  // st.shared (generic proxy) -> wgmma operand reads
        if (!__syncthreads_or(have)) continue;                // no neighbour in the chunk: exact zeros, nothing to add
        if constexpr (P == 3) {
            const uint64_t a_hi = make_desc_sw128(smem_u32(sa_hi)), a_lo = make_desc_sw128(smem_u32(sa_lo));
            const uint64_t b_hl = make_desc_sw128(smem_u32(sb));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < WT_CHUNK / MMA_K; ++k) {
                const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                wgmma_ss<2 * N>(acc, a_hi + koff, b_hl + koff, k == 0 ? 0u : 1u);
                wgmma_ss<N>(acc, a_lo + koff, b_hl + koff, 1);
            }
        } else {
            const uint64_t a_hi = make_desc_sw128(smem_u32(sa_hi)), b_hi = make_desc_sw128(smem_u32(sb));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < WT_CHUNK / MMA_K; ++k) {
                const uint64_t koff = (uint64_t)((k * MMA_K * ELEM_BYTES) >> 4);
                wgmma_ss<N>(acc, a_hi + koff, b_hi + koff, k == 0 ? 0u : 1u);
            }
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_operands<R>(acc);
        if constexpr (P == 3) {
#pragma unroll
            for (int j = 0; j < R / 2; ++j) sum[j] = __fadd_rn(__fadd_rn(sum[j], acc[j]), acc[R / 2 + j]);
        } else {
#pragma unroll
            for (int j = 0; j < R; ++j) sum[j] = __fadd_rn(sum[j], acc[j]);
        }
        __syncthreads();                                      // the next chunk overwrites the operand tiles
    }
    float *dst = partial + ((size_t)slab * num_kb + kb) * 64 * N;
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
        const int m = warp * 16 + (lane >> 2) + rh * 8;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2 *>(dst + (size_t)m * N + c) = make_float2(sum[4 * j + 2 * rh], sum[4 * j + 2 * rh + 1]);
        }
    }
}

__global__ void k_wgrad_tc_reduce(const float *__restrict__ partial, int num_kb, int pack, int K, int cin, int cout,
                                  const int *__restrict__ n_out_dev, int cap_out, const float *__restrict__ scale_dev,
                                  float *__restrict__ dw)
{
    const int n_out = min(*n_out_dev, cap_out);
    const int slabs = (n_out + WG_SLAB - 1) / WG_SLAB;
    const float sc = scale_dev ? __ldg(scale_dev) : 1.f;
    const long long elems = (long long)K * cin * cout;
    const size_t slab_elems = (size_t)num_kb * 64 * cout;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < elems;
         e += (long long)gridDim.x * blockDim.x) {
        const int co = (int)(e % cout), ci = (int)((e / cout) % cin), k = (int)(e / ((long long)cout * cin));
        const size_t src = ((size_t)(k / pack) * 64 + (size_t)(k % pack) * cin + ci) * cout + co;
        float s = 0.f;
        for (int j = 0; j < slabs; ++j) s += __ldg(&partial[(size_t)j * slab_elems + src]);
        dw[e] = scale_dev ? s * sc : s;
    }
}

template <int CIN, int COUT, int P>
int launch_wgrad_tc(const __half *x_hi, const __half *x_lo, int in_stride, const __half *g_hi, const __half *g_lo,
                    int g_stride, const int *nbr, int K, const int *n_out_dev, int cap_out, const int *perm,
                    const unsigned *tile_mask, float *partial, cudaStream_t stream)
{
    constexpr size_t smem = (P == 3 ? 2 : 1) * (64 * 128 + COUT * 128) + 1024;
    const int num_kb = (K + (64 / CIN) - 1) / (64 / CIN);
    k_wgrad_tc<CIN, COUT, P><<<dim3(num_slabs(cap_out), num_kb), WT_THREADS, smem, stream>>>(
        x_hi, x_lo, in_stride, g_hi, g_lo, g_stride, nbr, K, n_out_dev, cap_out, perm, tile_mask, partial);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

extern "C" size_t b2s_sparse_conv_wgrad_workspace_bytes(int cap_out, int K, int cin, int cout)
{
    if (cap_out <= 0 || K <= 0 || cin <= 0 || cout <= 0) return 0;
    return sizeof(float) * (size_t)num_slabs(cap_out) * K * cin * cout;
}

extern "C" int b2s_sparse_conv_wgrad(const float *feat_in, int cin, const float *dout, int cout, const int *nbr, int K,
                                     const int *num_out_dev, int cap_out, const float *scale_dev, float *dweight,
                                     void *workspace, size_t workspace_bytes, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(cin >= 1 && cout >= 1 && K >= 1 && K <= 65535 && cap_out >= 0, "b2s_sparse_conv_wgrad: bad sizes");
    B2S_REQUIRE(workspace_bytes >= b2s_sparse_conv_wgrad_workspace_bytes(cap_out, K, cin, cout),
                "b2s_sparse_conv_wgrad: workspace too small (b2s_sparse_conv_wgrad_workspace_bytes)");
    const long long elems = (long long)K * cin * cout;
    if (cap_out == 0) {
        B2S_CUDA_OK(cudaMemsetAsync(dweight, 0, sizeof(float) * elems, stream));
        return 0;
    }
    const int a = min((cin + 15) / 16, 4), b = min((cout + 15) / 16, 4);
    float *partial = reinterpret_cast<float *>(workspace);
#define B2S_WG_CASE(AA, BB) \
    if (a == AA && b == BB) launch_partial<AA, BB>(feat_in, cin, dout, cout, nbr, K, num_out_dev, cap_out, partial, stream);
    B2S_WG_CASE(1, 1) B2S_WG_CASE(1, 2) B2S_WG_CASE(1, 3) B2S_WG_CASE(1, 4)
    B2S_WG_CASE(2, 1) B2S_WG_CASE(2, 2) B2S_WG_CASE(2, 3) B2S_WG_CASE(2, 4)
    B2S_WG_CASE(3, 1) B2S_WG_CASE(3, 2) B2S_WG_CASE(3, 3) B2S_WG_CASE(3, 4)
    B2S_WG_CASE(4, 1) B2S_WG_CASE(4, 2) B2S_WG_CASE(4, 3) B2S_WG_CASE(4, 4)
#undef B2S_WG_CASE
    B2S_LAUNCH_OK();
    k_wgrad_reduce<<<grid_for(elems), kThreads, 0, stream>>>(partial, elems, num_out_dev, cap_out, scale_dev, dweight);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" size_t b2s_sparse_conv_wgrad_tc_workspace_bytes(int cap_out, int K, int cin, int cout)
{
    if (cap_out <= 0 || K <= 0 || cin <= 0 || cin > 64 || cout <= 0) return 0;
    const int pack = 64 / cin;
    return sizeof(float) * (size_t)num_slabs(cap_out) * ((K + pack - 1) / pack) * 64 * cout;
}

// products = 3: the 3xF16 form (b2s_sparse_conv_wgrad_tc).  products = 1: the f16 mode -- feat_lo and dout_lo must be
// NULL; X_hi^T * dY_hi, the same workspace.
extern "C" int b2s_sparse_conv_wgrad_tc_ex(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in,
                                           int cin, const b2s_half *dout_hi, const b2s_half *dout_lo, int dout_stride,
                                           int cout, const int *nbr, int K, const int *num_out_dev, int cap_out,
                                           const int *perm, const unsigned *tile_mask, const float *scale_dev,
                                           float *dweight, void *workspace, size_t workspace_bytes, int products,
                                           void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && feat_lo == nullptr && dout_lo == nullptr),
                "b2s_sparse_conv_wgrad_tc: products must be 3 (3xF16) or 1 (f16, no lo planes)");
    if (products == 1) { feat_lo = feat_hi; dout_lo = dout_hi; }   // (alignment checks below; never read)
    B2S_REQUIRE(b2s_sparse_conv_tc_supported(cin, cout),
                "b2s_sparse_conv_wgrad_tc: built for Cin in {8, 16, 32, 64}, Cout in {16, 32, 64} (others: "
                "b2s_sparse_conv_wgrad)");
    B2S_REQUIRE(K >= 1 && K <= 27 && cap_out >= 0 && rows_in >= 0, "b2s_sparse_conv_wgrad_tc: K must be 1..27");
    B2S_REQUIRE(in_stride >= cin && in_stride % 8 == 0 && dout_stride >= cout && dout_stride % 8 == 0 &&
                    ((uintptr_t)feat_hi & 15) == 0 && ((uintptr_t)feat_lo & 15) == 0 && ((uintptr_t)dout_hi & 15) == 0 &&
                    ((uintptr_t)dout_lo & 15) == 0,
                "b2s_sparse_conv_wgrad_tc: rows must be 16-byte aligned (strides multiples of 8 halves)");
    B2S_REQUIRE(workspace_bytes >= b2s_sparse_conv_wgrad_tc_workspace_bytes(cap_out, K, cin, cout),
                "b2s_sparse_conv_wgrad_tc: workspace too small (b2s_sparse_conv_wgrad_tc_workspace_bytes)");
    if (cap_out == 0) {
        B2S_CUDA_OK(cudaMemsetAsync(dweight, 0, sizeof(float) * (size_t)K * cin * cout, stream));
        return 0;
    }
    float *partial = reinterpret_cast<float *>(workspace);
    const __half *xh = reinterpret_cast<const __half *>(feat_hi), *xl = reinterpret_cast<const __half *>(feat_lo);
    const __half *gh = reinterpret_cast<const __half *>(dout_hi), *gl = reinterpret_cast<const __half *>(dout_lo);
    int rc = -2;
#define B2S_WT_CASE(CI, CO)                                                                                         \
    if (cin == CI && cout == CO)                                                                                    \
        rc = products == 1 ? launch_wgrad_tc<CI, CO, 1>(xh, nullptr, in_stride, gh, nullptr, dout_stride, nbr, K,    \
                                                        num_out_dev, cap_out, perm, tile_mask, partial, stream)      \
                           : launch_wgrad_tc<CI, CO, 3>(xh, xl, in_stride, gh, gl, dout_stride, nbr, K, num_out_dev, \
                                                        cap_out, perm, tile_mask, partial, stream);
    B2S_WT_CASE(64, 64) B2S_WT_CASE(64, 32) B2S_WT_CASE(64, 16) B2S_WT_CASE(32, 64) B2S_WT_CASE(32, 32)
    B2S_WT_CASE(32, 16) B2S_WT_CASE(16, 64) B2S_WT_CASE(16, 32) B2S_WT_CASE(16, 16) B2S_WT_CASE(8, 64)
    B2S_WT_CASE(8, 32) B2S_WT_CASE(8, 16)
#undef B2S_WT_CASE
    if (rc != 0) return rc;
    const int pack = 64 / cin;
    const long long elems = (long long)K * cin * cout;
    k_wgrad_tc_reduce<<<grid_for(elems), kThreads, 0, stream>>>(partial, (K + pack - 1) / pack, pack, K, cin, cout,
                                                                num_out_dev, cap_out, scale_dev, dweight);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_sparse_conv_wgrad_tc(const b2s_half *feat_hi, const b2s_half *feat_lo, int in_stride, int rows_in,
                                        int cin, const b2s_half *dout_hi, const b2s_half *dout_lo, int dout_stride,
                                        int cout, const int *nbr, int K, const int *num_out_dev, int cap_out,
                                        const int *perm, const unsigned *tile_mask, const float *scale_dev,
                                        float *dweight, void *workspace, size_t workspace_bytes, void *stream)
{
    return b2s_sparse_conv_wgrad_tc_ex(feat_hi, feat_lo, in_stride, rows_in, cin, dout_hi, dout_lo, dout_stride, cout,
                                       nbr, K, num_out_dev, cap_out, perm, tile_mask, scale_dev, dweight, workspace,
                                       workspace_bytes, 3, stream);
}

extern "C" int b2s_rulebook_transpose(const int *nbr, const int *num_out_dev, int cap_out, int K, int *nbrT, int cap_in,
                                      unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(K >= 1 && cap_out >= 0 && cap_in >= 0, "b2s_rulebook_transpose: bad sizes");
    if (cap_in > 0) B2S_CUDA_OK(cudaMemsetAsync(nbrT, 0xFF, sizeof(int) * (size_t)cap_in * K, stream));
    if (cap_out == 0) return 0;
    k_rulebook_transpose<<<grid_for((long long)cap_out * K), kThreads, 0, stream>>>(nbr, num_out_dev, cap_out, K, nbrT,
                                                                                  cap_in, status_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_from_bev(const float *dmap, const int *coors, const int *num_rows_dev, int cap_rows, int C, int batch,
                            int D, int H, int W, int layout, float *drows, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(C >= 1 && batch >= 1 && D >= 1 && H >= 1 && W >= 1 && cap_rows >= 0, "b2s_from_bev: bad sizes");
    B2S_REQUIRE(layout == B2S_LAYOUT_NCHW || layout == B2S_LAYOUT_NHWC, "b2s_from_bev: bad layout");
    if (cap_rows == 0) return 0;
    k_from_bev<<<grid_for((long long)cap_rows * C), kThreads, 0, stream>>>(dmap, coors, num_rows_dev, cap_rows, C, batch,
                                                                          D, H, W, layout, drows);
    B2S_LAUNCH_OK();
    return 0;
}

// products = 1: lo must be NULL, only the hi plane is written (the same bits as the hi plane of products = 3)
extern "C" int b2s_split_f16_autoscale_ex(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev,
                                          int cap_rows, int row_floats, int out_channels, int out_stride,
                                          float *scale_dev, int products, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && lo == nullptr),
                "b2s_split_f16_autoscale: products must be 3 (hi/lo planes) or 1 (f16, no lo plane)");
    B2S_REQUIRE(row_floats >= 1 && out_channels >= row_floats && out_channels % 8 == 0 && out_stride >= out_channels &&
                    out_stride % 8 == 0 && cap_rows >= 0,
                "b2s_split_f16_autoscale: out_channels / out_stride must be multiples of 8, out_stride >= out_channels >= "
                "row_floats");
    B2S_REQUIRE(((uintptr_t)hi & 15) == 0 && ((uintptr_t)lo & 15) == 0,
                "b2s_split_f16_autoscale: planes must be 16-byte aligned");
    B2S_REQUIRE(scale_dev != nullptr, "b2s_split_f16_autoscale: scale_dev is required");
    B2S_CUDA_OK(cudaMemsetAsync(scale_dev + 1, 0, sizeof(float), stream));
    const long long n = (long long)cap_rows * row_floats;
    if (n > 0) {
        k_absmax<<<grid_for(n), kThreads, 0, stream>>>(x, num_rows_dev, cap_rows, row_floats,
                                                      reinterpret_cast<unsigned *>(scale_dev + 1));
        B2S_LAUNCH_OK();
    }
    // one CTA at least: it writes scale_dev[0] even when there are no rows
    if (products == 1)
        k_split_f16_scaled<1><<<grid_for((long long)cap_rows * (out_channels / 8)), kThreads, 0, stream>>>(
            x, reinterpret_cast<__half *>(hi), nullptr, num_rows_dev, cap_rows, row_floats, out_channels, out_stride,
            scale_dev);
    else
        k_split_f16_scaled<3><<<grid_for((long long)cap_rows * (out_channels / 8)), kThreads, 0, stream>>>(
            x, reinterpret_cast<__half *>(hi), reinterpret_cast<__half *>(lo), num_rows_dev, cap_rows, row_floats,
            out_channels, out_stride, scale_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_split_f16_autoscale(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows,
                                       int row_floats, int out_channels, int out_stride, float *scale_dev, void *stream)
{
    return b2s_split_f16_autoscale_ex(x, hi, lo, num_rows_dev, cap_rows, row_floats, out_channels, out_stride, scale_dev,
                                      3, stream);
}

// products = 1: lo must be NULL, only the hi plane is written (the same bits as the hi plane of products = 3)
extern "C" int b2s_pack_sparse_weights_ex(const float *w, int K, int cin, int cout, int transpose, int flip, b2s_half *hi,
                                          b2s_half *lo, float *scale_dev, int products, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && lo == nullptr),
                "b2s_pack_sparse_weights: products must be 3 (hi/lo planes) or 1 (f16, no lo plane)");
    if (products == 1) lo = hi;                       // (the checks below; never written)
    const int n_in = transpose ? cout : cin, n_out = transpose ? cin : cout;
    const int n_in_pad = n_in <= 8 ? 8 : n_in;
    B2S_REQUIRE(K >= 1 && cin >= 1 && cout >= 1 && n_in >= 1 && (n_in_pad == 8 || n_in_pad == 16 || n_in_pad == 32 ||
                                                                  n_in_pad == 64),
                "b2s_pack_sparse_weights: the packed input channels must be 1..8, 16, 32 or 64 (got %d)", n_in);
    B2S_REQUIRE(transpose == 0 || transpose == 1, "b2s_pack_sparse_weights: transpose must be 0 or 1");
    B2S_REQUIRE(w && hi && lo && scale_dev, "b2s_pack_sparse_weights: w, hi, lo and scale_dev required");
    B2S_REQUIRE(((uintptr_t)hi & 15) == 0 && ((uintptr_t)lo & 15) == 0,
                "b2s_pack_sparse_weights: planes must be 16-byte aligned");
    const int pack = b2s_tc::BLOCK_K / n_in_pad, nkb = (K + pack - 1) / pack;
    const long long n = (long long)K * cin * cout;
    B2S_REQUIRE(n < (1ll << 31), "b2s_pack_sparse_weights: weight too large");
    B2S_CUDA_OK(cudaMemsetAsync(scale_dev + 2, 0, sizeof(float), stream));
    k_absmax<<<grid_for(n), kThreads, 0, stream>>>(w, nullptr, 1, (int)n, reinterpret_cast<unsigned *>(scale_dev + 2));
    B2S_LAUNCH_OK();
    if (products == 1)
        k_pack_sparse_weights<1><<<grid_for((long long)nkb * n_out * (b2s_tc::BLOCK_K / 8)), kThreads, 0, stream>>>(
            w, K, cin, cout, transpose, flip ? 1 : 0, n_in, n_in_pad, n_out, nkb, reinterpret_cast<__half *>(hi), nullptr,
            scale_dev);
    else
        k_pack_sparse_weights<3><<<grid_for((long long)nkb * n_out * (b2s_tc::BLOCK_K / 8)), kThreads, 0, stream>>>(
            w, K, cin, cout, transpose, flip ? 1 : 0, n_in, n_in_pad, n_out, nkb, reinterpret_cast<__half *>(hi),
            reinterpret_cast<__half *>(lo), scale_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_pack_sparse_weights(const float *w, int K, int cin, int cout, int transpose, int flip, b2s_half *hi,
                                       b2s_half *lo, float *scale_dev, void *stream)
{
    return b2s_pack_sparse_weights_ex(w, K, cin, cout, transpose, flip, hi, lo, scale_dev, 3, stream);
}

// products = 1: lo must be NULL, only the hi plane is written (the same bits as the hi plane of products = 3)
extern "C" int b2s_pack_conv2d_weights_ex(const float *w, int cout, int cin, int transpose, b2s_half *hi, b2s_half *lo,
                                          float *scale_dev, int products, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && lo == nullptr),
                "b2s_pack_conv2d_weights: products must be 3 (hi/lo planes) or 1 (f16, no lo plane)");
    if (products == 1) lo = hi;                       // (the checks below; never written)
    B2S_REQUIRE(cout >= 1 && cin >= 1 && cout % 64 == 0 && cin % 64 == 0,
                "b2s_pack_conv2d_weights: cin and cout must be multiples of 64");
    B2S_REQUIRE(transpose == 0 || transpose == 1, "b2s_pack_conv2d_weights: transpose must be 0 or 1");
    B2S_REQUIRE(w && hi && lo && scale_dev, "b2s_pack_conv2d_weights: w, hi, lo and scale_dev required");
    B2S_REQUIRE(((uintptr_t)hi & 15) == 0 && ((uintptr_t)lo & 15) == 0,
                "b2s_pack_conv2d_weights: planes must be 16-byte aligned");
    const long long n = 9ll * cin * cout;
    B2S_REQUIRE(n < (1ll << 31), "b2s_pack_conv2d_weights: weight too large");
    const int n_in = transpose ? cout : cin, n_out = transpose ? cin : cout;
    const int n_pad = n_out < 128 ? n_out : 128, groups = (n_out + 127) / 128;
    B2S_CUDA_OK(cudaMemsetAsync(scale_dev + 2, 0, sizeof(float), stream));
    k_absmax<<<grid_for(n), kThreads, 0, stream>>>(w, nullptr, 1, (int)n, reinterpret_cast<unsigned *>(scale_dev + 2));
    B2S_LAUNCH_OK();
    if (products == 1)
        k_pack_conv2d_weights<1><<<grid_for((long long)groups * 9 * n_pad * (n_in / 8)), kThreads, 0, stream>>>(
            w, cout, cin, transpose, n_in, n_out, n_pad, groups, reinterpret_cast<__half *>(hi), nullptr, scale_dev);
    else
        k_pack_conv2d_weights<3><<<grid_for((long long)groups * 9 * n_pad * (n_in / 8)), kThreads, 0, stream>>>(
            w, cout, cin, transpose, n_in, n_out, n_pad, groups, reinterpret_cast<__half *>(hi),
            reinterpret_cast<__half *>(lo), scale_dev);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_pack_conv2d_weights(const float *w, int cout, int cin, int transpose, b2s_half *hi, b2s_half *lo,
                                       float *scale_dev, void *stream)
{
    return b2s_pack_conv2d_weights_ex(w, cout, cin, transpose, hi, lo, scale_dev, 3, stream);
}
