// tc_util.cu -- conversions between fp32 rows and the fp16 hi/lo planes (3xF16 split, tc_common.cuh) the
// tensor-core kernels consume.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace {

// one thread per (row, 8-channel group of the OUTPUT row): reads up to 8 floats, writes 16 bytes per plane (P = 1: the
// hi plane only)
template <int P>
__global__ void k_split_f16(const float *__restrict__ x, __half *__restrict__ hi, __half *__restrict__ lo,
                            const int *__restrict__ n_rows_dev, int cap_rows, int row_floats, int out_channels,
                            int out_stride)
{
    const int groups = out_channels / 8;
    const long long n = (long long)(n_rows_dev ? min(*n_rows_dev, cap_rows) : cap_rows) * groups;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / groups;
        const int c0 = (int)(i - row * groups) * 8;
        uint32_t h[4], l[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = c0 + 2 * j;
            const float a = c < row_floats ? __ldg(&x[row * row_floats + c]) : 0.f;        // channels past the input
            const float b = c + 1 < row_floats ? __ldg(&x[row * row_floats + c + 1]) : 0.f;  // row are zero padding
            const uint32_t pa = b2s_tc::split_f16(a), pb = b2s_tc::split_f16(b);
            h[j] = __byte_perm(pa, pb, 0x5410);
            l[j] = __byte_perm(pa, pb, 0x7632);
        }
        *reinterpret_cast<uint4 *>(hi + row * out_stride + c0) = make_uint4(h[0], h[1], h[2], h[3]);
        if constexpr (P == 3) *reinterpret_cast<uint4 *>(lo + row * out_stride + c0) = make_uint4(l[0], l[1], l[2], l[3]);
    }
}

__global__ void k_merge_f16(const __half *__restrict__ hi, const __half *__restrict__ lo, float *__restrict__ x,
                            const int *__restrict__ n_rows_dev, int cap_rows, int row_floats, int in_stride)
{
    const int pairs = row_floats / 2;
    const long long n = (long long)(n_rows_dev ? min(*n_rows_dev, cap_rows) : cap_rows) * pairs;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / pairs;
        const int c = (int)(i - row * pairs) * 2;
        const float2 h = __half22float2(*reinterpret_cast<const __half2 *>(hi + row * in_stride + c));
        const float2 l = __half22float2(*reinterpret_cast<const __half2 *>(lo + row * in_stride + c));
        *reinterpret_cast<float2 *>(x + row * row_floats + c) = make_float2(h.x + l.x, h.y + l.y);   // exact in fp32
    }
}

inline int grid_for(long long items)
{
    long long b = (items + 255) / 256;
    return (int)(b < 1 ? 1 : (b < 132 * 8 ? b : 132 * 8));
}

}  // namespace

// x [rows, row_floats] fp32 -> hi = fp16(x), lo = fp16(x - hi): out_channels halves per row and plane (>= row_floats,
// multiple of 8; columns past row_floats are written as zeros), rows out_stride halves apart (>= out_channels,
// multiple of 8 -- e.g. 2*out_channels for interleaved [row][hi | lo] storage).  rows = *num_rows_dev (NULL: cap_rows).
// products = 1 (the f16 mode): lo must be NULL, only hi = fp16(x) is written.
extern "C" int b2s_split_f16_ex(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows,
                                int row_floats, int out_channels, int out_stride, int products, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(products == 3 || (products == 1 && lo == nullptr),
                "b2s_split_f16: products must be 3 (hi/lo planes) or 1 (f16, no lo plane)");
    B2S_REQUIRE(row_floats >= 1 && out_channels >= row_floats && out_channels % 8 == 0 && out_stride >= out_channels &&
                    out_stride % 8 == 0 && cap_rows >= 0,
                "b2s_split_f16: out_channels / out_stride must be multiples of 8, out_stride >= out_channels >= row_floats");
    B2S_REQUIRE(((uintptr_t)hi & 15) == 0 && ((uintptr_t)lo & 15) == 0, "b2s_split_f16: planes must be 16-byte aligned");
    const long long items = (long long)cap_rows * (out_channels / 8);
    if (items == 0) return 0;
    if (products == 1)
        k_split_f16<1><<<grid_for(items), 256, 0, stream>>>(x, reinterpret_cast<__half *>(hi), nullptr, num_rows_dev,
                                                            cap_rows, row_floats, out_channels, out_stride);
    else
        k_split_f16<3><<<grid_for(items), 256, 0, stream>>>(x, reinterpret_cast<__half *>(hi),
                                                            reinterpret_cast<__half *>(lo), num_rows_dev, cap_rows,
                                                            row_floats, out_channels, out_stride);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_split_f16(const float *x, b2s_half *hi, b2s_half *lo, const int *num_rows_dev, int cap_rows,
                             int row_floats, int out_channels, int out_stride, void *stream)
{
    return b2s_split_f16_ex(x, hi, lo, num_rows_dev, cap_rows, row_floats, out_channels, out_stride, 3, stream);
}

// hi/lo rows of in_stride halves -> x [rows, row_floats] fp32 = hi + lo (exact).  row_floats even.
extern "C" int b2s_merge_f16(const b2s_half *hi, const b2s_half *lo, float *x, const int *num_rows_dev, int cap_rows,
                             int row_floats, int in_stride, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(row_floats >= 2 && row_floats % 2 == 0 && in_stride >= row_floats && in_stride % 2 == 0 && cap_rows >= 0,
                "b2s_merge_f16: row_floats and in_stride must be even, in_stride >= row_floats");
    const long long items = (long long)cap_rows * (row_floats / 2);
    if (items == 0) return 0;
    k_merge_f16<<<grid_for(items), 256, 0, stream>>>(reinterpret_cast<const __half *>(hi),
                                                     reinterpret_cast<const __half *>(lo), x, num_rows_dev, cap_rows,
                                                     row_floats, in_stride);
    B2S_LAUNCH_OK();
    return 0;
}
