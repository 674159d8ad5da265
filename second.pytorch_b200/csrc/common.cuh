// common.cuh -- shared helpers for libb2second.so (sm_90a).  See include/b2second.h for the ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "b2second.h"

#define B2S_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull
#define B2S_INF_IDX 0x7F7F7F7F  // what cudaMemsetAsync(..., 0x7F, ...) writes into an int32

void b2s_set_error(const char *fmt, ...);

#define B2S_CUDA_OK(expr)                                                              \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess) {                                                       \
            b2s_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,                 \
                          cudaGetErrorString(_e));                                     \
            return -1;                                                                 \
        }                                                                              \
    } while (0)

#define B2S_LAUNCH_OK()                                                                \
    do {                                                                               \
        cudaError_t _e = cudaPeekAtLastError();                                        \
        if (_e != cudaSuccess) {                                                       \
            b2s_set_error("%s:%d kernel launch -> %s", __FILE__, __LINE__,             \
                          cudaGetErrorString(_e));                                     \
            return -1;                                                                 \
        }                                                                              \
    } while (0)

#define B2S_REQUIRE(cond, ...)                                                         \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            b2s_set_error(__VA_ARGS__);                                                \
            return -2;                                                                 \
        }                                                                              \
    } while (0)

static inline int b2s_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline size_t b2s_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// 64-bit mix (murmur3 finaliser) -> table slot
__device__ __forceinline__ uint32_t b2s_hash64(unsigned long long k)
{
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (uint32_t)k;
}

__device__ __forceinline__ unsigned long long b2s_flat_key(int b, int z, int y, int x, int D, int H,
                                                           int W)
{
    return (((unsigned long long)b * D + z) * H + y) * (unsigned long long)W + x;
}

// open addressing, linear probing.  returns slot index, or -1 when the table is full.
__device__ __forceinline__ int b2s_hash_insert(unsigned long long *keys, int mask,
                                               unsigned long long key)
{
    uint32_t h = b2s_hash64(key) & (uint32_t)mask;
    for (int probe = 0; probe <= mask; ++probe) {
        unsigned long long prev = atomicCAS(&keys[h], B2S_EMPTY_KEY, key);
        if (prev == B2S_EMPTY_KEY || prev == key) return (int)h;
        h = (h + 1) & (uint32_t)mask;
    }
    return -1;
}

// returns the value stored for key, or -1
__device__ __forceinline__ int b2s_hash_find(const unsigned long long *__restrict__ keys,
                                             const int *__restrict__ vals, int mask,
                                             unsigned long long key)
{
    uint32_t h = b2s_hash64(key) & (uint32_t)mask;
    for (int probe = 0; probe <= mask; ++probe) {
        unsigned long long k = __ldg(&keys[h]);
        if (k == key) return __ldg(&vals[h]);
        if (k == B2S_EMPTY_KEY) return -1;
        h = (h + 1) & (uint32_t)mask;
    }
    return -1;
}

// block-wide exclusive scan of one int per thread (blockDim.x multiple of 32, <= 1024).
// returns the exclusive prefix; *total (same for all threads) = block sum.
__device__ __forceinline__ int b2s_block_exscan(int v, int *total)
{
    __shared__ int s_warp_sum[32];
    __shared__ int s_warp_off[32];
    __shared__ int s_total;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int nw = (blockDim.x + 31) >> 5;
    __syncthreads();  // protect the shared arrays when called back to back
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp_sum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        int s = lane < nw ? s_warp_sum[lane] : 0;
        int si = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, si, o);
            if (lane >= o) si += t;
        }
        s_warp_off[lane] = si - s;
        if (lane == 31) s_total = si;
    }
    __syncthreads();
    *total = s_total;
    return inc - v + s_warp_off[wid];
}
