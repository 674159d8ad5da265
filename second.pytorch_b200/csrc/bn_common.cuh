// bn_common.cuh -- the train-mode BatchNorm steps shared by the PointPillars feature net (pfn_train.cu) and the
// BatchNorm + ReLU pair (bn_train.cu), so both update the running buffers and derive their factors the same way.
#pragma once
#include "common.cuh"

// s = 1 / sqrt(var + eps), in float64
__device__ __forceinline__ double b2s_bn_inv_std(double var, float eps) { return 1.0 / sqrt(var + (double)eps); }

// the running buffers of channel c, as torch's CUDA BatchNorm updates them: fp32, rm = m * mean + (1 - m) * rm and
// rv = m * var * M / (M - 1) + (1 - m) * rv (the batch variance unbiased), every step rounded on its own
__device__ __forceinline__ void b2s_bn_update_running(float *rmean, float *rvar, int c, double mean, double var,
                                                      double M, float momentum)
{
    const float m32 = (float)mean, uv32 = (float)(var * (M / (M - 1.0)));
    const float keep = __fsub_rn(1.f, momentum);
    rmean[c] = __fadd_rn(__fmul_rn(momentum, m32), __fmul_rn(keep, rmean[c]));
    rvar[c] = __fadd_rn(__fmul_rn(momentum, uv32), __fmul_rn(keep, rvar[c]));
}
