// autoscale.cuh -- the device-side power-of-two scale of the 3xF16 split (b2second/tc.py: pow2_scale): max|x| as an
// order-independent integer reduction and the exponent rule.  Shared by the sparse training path (sparse_grad.cu) and
// the dense RPN training path (conv_train.cu), so both pick bit-identical scales.
#pragma once
#include "common.cuh"

namespace {

// max |x| over the finite elements of the live rows as the bit pattern of a non-negative float (ordered like unsigned
// ints): integer atomicMax, so the result does not depend on the order.  Inf and NaN are left out, so one non-finite
// element does not take the scale of all the others (the splits carry it through as itself: split_f16_keep_nonfinite).
__global__ void k_absmax(const float *__restrict__ x, const int *__restrict__ n_rows_dev, int cap_rows, int row_floats,
                         unsigned *__restrict__ amax_bits)
{
    const long long n = (long long)(n_rows_dev ? min(*n_rows_dev, cap_rows) : cap_rows) * row_floats;
    unsigned m = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const unsigned b = __float_as_uint(__ldg(&x[i])) & 0x7FFFFFFFu;
        if (b < 0x7F800000u) m = max(m, b);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(amax_bits, m);
}

// e with max|x| * 2^e in (2^12, 2^13] (b2second/tc.py: pow2_scale, which also clamps as autoscale_exponent does), 0 for
// zero or non-finite max|x|
__device__ __forceinline__ int pow2_exponent(unsigned amax_bits)
{
    const float m = __uint_as_float(amax_bits);
    if (amax_bits == 0 || amax_bits >= 0x7F800000u) return 0;
    int ex;
    const float f = frexpf(m, &ex);                 // m = f * 2^ex, f in [0.5, 1)
    const int ceil_log2 = f == 0.5f ? ex - 1 : ex;
    return 13 - ceil_log2;
}

// pow2_exponent clamped so that 2^e and 2^-e are normal floats (max|x| below 2^-113 would otherwise give 2^e = inf)
__device__ __forceinline__ int autoscale_exponent(unsigned amax_bits)
{
    return min(max(pow2_exponent(amax_bits), -126), 126);
}

}  // namespace
