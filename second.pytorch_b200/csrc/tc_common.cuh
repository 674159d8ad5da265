// tc_common.cuh -- wgmma / TMA / mbarrier helpers shared by the tensor-core kernels (sm_90a).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace b2s_tc {

// Operand format ("3xF16"): every fp32 operand x is carried as two fp16 planes, hi = fp16_rn(x) and
// lo = fp16_rn(x - hi): 22 significand bits while lo is a normal fp16, 2^-25 absolute otherwise (fp16 subnormals are
// exact operands for the tensor core).  Each K step issues A_hi*B_hi + A_hi*B_lo + A_lo*B_hi with fp32 accumulation in
// registers (the dropped lo*lo term is ~2^-22 relative) -- the same three products as a 3xTF32 split, but f16 MMAs
// run at twice the tf32 rate and the planes are half the bytes.  Weights are pre-scaled by a power of two
// per layer (folded into the epilogue scale) so that their lo plane stays in the normal range
// (b2second/tc.py: split_f16); activations are stored unscaled (|x| <= 65504, saturating conversion).
constexpr int BLOCK_M = 128;   // rows of an A tile (two warpgroups of 64)
constexpr int BLOCK_K = 64;    // 64 fp16 = 128 B = one SWIZZLE_128B row
constexpr int MMA_K = 16;      // f16: 32 bytes per MMA K step
constexpr int ELEM_BYTES = 2;
constexpr uint32_t A_TILE_BYTES = BLOCK_M * BLOCK_K * ELEM_BYTES;   // 16 KB

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// warp index as a warp-uniform value (role dispatch without divergence inside a warp)
__device__ __forceinline__ int warp_idx_uniform() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bounded wait: ~seconds of spinning, then trap (a protocol bug must not hang the device)
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t addr = smem_u32(bar);
    // not unrolled: the compiler otherwise replicates the try_wait ~60x at every call site, and these warp-specialised
    // kernels (several roles = several instruction streams per SM) are sensitive to instruction-cache footprint
#pragma unroll 1
    for (uint32_t it = 0; it < (1u << 28); ++it) {
        uint32_t done;
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return;
    }
    __trap();
}

__device__ __forceinline__ void tma_load_4d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1,
                                            int c2, int c3)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap *map, int c0, int c1, int c2, int c3)
{
    asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global [%0, {%1, %2, %3, %4}];" ::"l"(map), "r"(c0), "r"(c1),
                 "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *smem_dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1,
                                            int c2)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma): 8-row groups 1024 B apart.  Advancing K by 16
// fp16 elements inside the 128-byte swizzle row adds 32 B (2 in the 16-byte address field).
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);        // start address, 16-byte units
    d |= (uint64_t)1 << 16;                            // leading byte offset (unused for swizzled K-major): 1
    d |= (uint64_t)(1024 >> 4) << 32;                  // stride byte offset between 8-row groups
    d |= (uint64_t)1 << 62;                            // layout type: SWIZZLE_128B
    return d;
}

// ---- warpgroup MMA (wgmma, sm_90a): D[64 rows, N] (+)= A[64, 16] * B[N, 16]^T, fp16 operands, fp32 accumulators in
// registers.  Accumulator fragment of thread t of the warpgroup (warp w = t / 32, lane l): for every 8-column block j,
// d[4j + 0/1] = row 16w + l/4, columns 8j + 2(l%4) + 0/1, and d[4j + 2/3] = the same columns of row 16w + l/4 + 8.
// scale_d = 0 overwrites the accumulators (first product of an accumulation chain).
template <int N> __device__ __forceinline__ void wgmma_ss(float *d, uint64_t da, uint64_t db, uint32_t scale_d);
// A operand from registers: the fragment of a 64x16 fp16 tile, a[0] = (row 16w + l/4, k 2(l%4) + 0/1), a[1] = row + 8,
// a[2] / a[3] = the same rows at k + 8 -- exactly the accumulator fragment of a 16-column block pair, packed to fp16.
template <int N> __device__ __forceinline__ void wgmma_rs(float *d, const uint32_t *a, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_ss<16>(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<32>(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<32>(float *d, const uint32_t *a, uint64_t db, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<64>(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<128>(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// pins the accumulator registers after a wait: the compiler must not read them before the wgmma that writes them retired
template <int R> __device__ __forceinline__ void wgmma_fence_operands(float *d)
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// generic-proxy writes to shared memory (cp.async, st.shared) -> visible to the wgmma operand reads (async proxy)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// fp32 -> (hi, lo) fp16 pair packed in one register: hi in bits 0-15, lo in bits 16-31.  Saturating conversions
// (a value beyond +-65504 clamps instead of turning into inf and poisoning the accumulators).
__device__ __forceinline__ uint32_t split_f16(float v)
{
    uint16_t h, l;
    float hf;
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    asm("cvt.f32.f16 %0, %1;" : "=f"(hf) : "h"(h));
    asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(l) : "f"(v - hf));
    return (uint32_t)h | ((uint32_t)l << 16);
}
// the split of the automatically scaled paths (training inputs, gradients, weight packs): v is x * 2^e with
// max|x_finite| * 2^e <= 2^13, so a finite v never needs the saturation.  A non-finite v stays itself in hi (+-inf, NaN)
// with lo = +0, so it reaches the result as torch's fp32 arithmetic would carry it.
__device__ __forceinline__ uint32_t split_f16_keep_nonfinite(float v)
{
    uint16_t h, l;
    float hf;
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(v));
    asm("cvt.f32.f16 %0, %1;" : "=f"(hf) : "h"(h));
    asm("cvt.rn.f16.f32 %0, %1;" : "=h"(l) : "f"(isfinite(v) ? v - hf : 0.f));
    return (uint32_t)h | ((uint32_t)l << 16);
}
__device__ __forceinline__ float f16_bits_to_float(uint16_t h)
{
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    return f;
}


// ---- host side: per-device caches (a process may drive several GPUs: SM count and the opt-in dynamic shared memory
// attribute belong to the CURRENT device, so they are cached per device index, not in a process-wide static) ----
constexpr int kMaxDevices = 64;
inline int current_device()
{
    int d = 0;
    cudaGetDevice(&d);
    return d & (kMaxDevices - 1);
}
inline int num_sms_current()
{
    static int sms[kMaxDevices] = {0};
    const int d = current_device();
    if (!sms[d]) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || v <= 0) v = 132;
        sms[d] = v;
    }
    return sms[d];
}
// opt a kernel into `bytes` of dynamic shared memory on the current device (once per device and kernel instance)
#define B2S_SMEM_OPT_IN(kernel, bytes)                                                                           \
    do {                                                                                                         \
        static bool _done[b2s_tc::kMaxDevices] = {false};                                                        \
        const int _d = b2s_tc::current_device();                                                                 \
        if (!_done[_d]) {                                                                                        \
            B2S_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
            _done[_d] = true;                                                                                    \
        }                                                                                                        \
    } while (0)

// ---- host side: tensor maps through the driver entry point (no link-time libcuda dependency) ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode()
{
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
        return nullptr;
    fn = (PFN_encodeTiled)p;
    return fn;
}

// elem_strides (optional): traversal stride per dimension -- {1, s, s, 1} fetches every s-th pixel (strided conv)
inline int make_map(CUtensorMap *m, const void *base, int rank, const cuuint64_t *dims,
                    const cuuint64_t *strides_bytes, const cuuint32_t *box, const cuuint32_t *elem_strides = nullptr)
{
    PFN_encodeTiled enc = get_encode();
    if (!enc) { b2s_set_error("cuTensorMapEncodeTiled entry point not available"); return -1; }
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    if (elem_strides)
        for (int i = 0; i < rank; ++i) estr[i] = elem_strides[i];
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, (void *)base, dims, strides_bytes, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { b2s_set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return -1; }
    return 0;
}

}  // namespace b2s_tc
