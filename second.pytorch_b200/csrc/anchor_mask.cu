// anchor_mask.cu -- the anchor-area mask of the reference's preprocessing (second/data/preprocess.py:345-357):
//   count map        box_np_ops.sparse_sum_for_anchors_mask (box_np_ops.py:917-922): voxels per BEV cell (b, y, x)
//   summed-area      dense_voxel_map.cumsum(0).cumsum(1): inclusive prefix sums along x, then along y, per frame
//   per-anchor area  box_np_ops.fused_get_anchors_area (box_np_ops.py:925-946) over host-derived integer boxes,
//                    mask = area > threshold
// The reference holds the map in float32; every value is an integer below 2^24 (at most one frame's voxel count), so
// the int32 map here equals it bit for bit and the integer atomics make the count order-independent.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kColUnroll = 8;

// one integer atomicAdd per surviving voxel at (b, y, x); coordinates outside the map are ignored
__global__ void __launch_bounds__(kThreads)
k_am_scatter(const int *__restrict__ coors, const int *__restrict__ num_dev, int cap, int B, int ny, int nx,
             int *__restrict__ map)
{
    const int i = blockIdx.x * kThreads + threadIdx.x;
    int n = __ldg(num_dev);
    n = n < cap ? n : cap;
    if (i >= n) return;
    const int4 c = __ldg(reinterpret_cast<const int4 *>(coors) + i);     // (b, z, y, x)
    if ((unsigned)c.x >= (unsigned)B || (unsigned)c.z >= (unsigned)ny || (unsigned)c.w >= (unsigned)nx) return;
    atomicAdd(&map[((size_t)c.x * ny + c.z) * nx + c.w], 1);
}

// inclusive scan along x: one warp per row (b, y), 32 cells per step with the carry in a register
__global__ void __launch_bounds__(kThreads)
k_am_scan_rows(int *__restrict__ map, int rows, int nx)
{
    const int row = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    int *r = map + (size_t)row * nx;
    int carry = 0;
    for (int x0 = 0; x0 < nx; x0 += 32) {
        const int x = x0 + lane;
        int v = x < nx ? r[x] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += t;
        }
        v += carry;
        if (x < nx) r[x] = v;
        carry = __shfl_sync(0xffffffffu, v, 31);
    }
}

// inclusive scan along y: one thread per column (b, x), consecutive threads on consecutive x (coalesced rows);
// kColUnroll rows are loaded before they are added so that many loads are in flight per thread
__global__ void __launch_bounds__(kThreads)
k_am_scan_cols(int *__restrict__ map, int B, int ny, int nx)
{
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= B * nx) return;
    const int b = i / nx, x = i - b * nx;
    int *col = map + (size_t)b * ny * nx + x;
    int acc = 0;
    int y = 0;
    for (; y + kColUnroll <= ny; y += kColUnroll) {
        int v[kColUnroll];
#pragma unroll
        for (int k = 0; k < kColUnroll; ++k) v[k] = col[(size_t)(y + k) * nx];
#pragma unroll
        for (int k = 0; k < kColUnroll; ++k) {
            acc += v[k];
            col[(size_t)(y + k) * nx] = acc;
        }
    }
    for (; y < ny; ++y) {
        acc += col[(size_t)y * nx];
        col[(size_t)y * nx] = acc;
    }
}

// one thread per (frame, anchor): area = S[y1,x1] - S[y1,x0] - S[y0,x1] + S[y0,x0] over the half-open box
// (x0, x1] x (y0, y1] exactly as fused_get_anchors_area reads it (no -1 on the low corner)
__global__ void __launch_bounds__(kThreads)
k_am_lookup(const int *__restrict__ map, int B, int ny, int nx, const int4 *__restrict__ boxes, int A, float threshold,
            uint8_t *__restrict__ mask)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= (long long)B * A) return;
    const int b = (int)(i / A), a = (int)(i - (long long)b * A);
    int4 bx = __ldg(boxes + a);                                            // (x0, y0, x1, y1)
    // the host validated 0 <= x0 <= x1 < nx, 0 <= y0 <= y1 < ny; clamping keeps a bad buffer from reading outside
    bx.x = min(max(bx.x, 0), nx - 1);
    bx.z = min(max(bx.z, 0), nx - 1);
    bx.y = min(max(bx.y, 0), ny - 1);
    bx.w = min(max(bx.w, 0), ny - 1);
    const int *S = map + (size_t)b * ny * nx;
    const int ID = __ldg(S + (size_t)bx.w * nx + bx.z);
    const int IA = __ldg(S + (size_t)bx.y * nx + bx.x);
    const int IB = __ldg(S + (size_t)bx.w * nx + bx.x);
    const int IC = __ldg(S + (size_t)bx.y * nx + bx.z);
    const int area = ID - IB - IC + IA;
    mask[i] = (float)area > threshold ? 1 : 0;
}

}  // namespace

extern "C" size_t b2s_anchor_area_mask_workspace_bytes(int batch, int ny, int nx)
{
    if (batch <= 0 || ny <= 0 || nx <= 0) return 0;
    return sizeof(int) * (size_t)batch * (size_t)ny * (size_t)nx;
}

extern "C" int b2s_anchor_area_mask(const int *coors, const int *num_dev, int cap, int batch, int ny, int nx,
                                    const int *anchor_boxes, int num_anchors, float threshold, void *count_map_ws,
                                    size_t workspace_bytes, uint8_t *mask_out, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && ny >= 1 && nx >= 1, "b2s_anchor_area_mask: batch, ny and nx must be >= 1");
    B2S_REQUIRE(cap >= 0 && cap < (1 << 24), "b2s_anchor_area_mask: cap must be in [0, 2^24) (exact float32 counts)");
    B2S_REQUIRE(num_anchors >= 0, "b2s_anchor_area_mask: num_anchors must be >= 0");
    B2S_REQUIRE((size_t)batch * ny * nx < ((size_t)1 << 31), "b2s_anchor_area_mask: count map above 2^31 cells");
    B2S_REQUIRE(count_map_ws != nullptr && workspace_bytes >= b2s_anchor_area_mask_workspace_bytes(batch, ny, nx),
                "b2s_anchor_area_mask: workspace too small");
    B2S_REQUIRE(cap == 0 || (coors != nullptr && num_dev != nullptr), "b2s_anchor_area_mask: coors and num_dev required");
    B2S_REQUIRE(((uintptr_t)coors & 15) == 0, "b2s_anchor_area_mask: coors must be 16-byte aligned int32 [cap, 4] rows");
    B2S_REQUIRE(num_anchors == 0 || (anchor_boxes != nullptr && mask_out != nullptr && ((uintptr_t)anchor_boxes & 15) == 0),
                "b2s_anchor_area_mask: anchor_boxes (16-byte aligned int32 [A, 4]) and mask_out required");
    int *map = (int *)count_map_ws;
    const size_t cells = (size_t)batch * ny * nx;
    B2S_CUDA_OK(cudaMemsetAsync(map, 0, sizeof(int) * cells, stream));
    if (cap > 0) {
        k_am_scatter<<<b2s_cdiv(cap, kThreads), kThreads, 0, stream>>>(coors, num_dev, cap, batch, ny, nx, map);
        B2S_LAUNCH_OK();
    }
    const int rows = batch * ny;
    k_am_scan_rows<<<b2s_cdiv(rows, kThreads / 32), kThreads, 0, stream>>>(map, rows, nx);
    B2S_LAUNCH_OK();
    k_am_scan_cols<<<b2s_cdiv((long long)batch * nx, kThreads), kThreads, 0, stream>>>(map, batch, ny, nx);
    B2S_LAUNCH_OK();
    if (num_anchors > 0) {
        k_am_lookup<<<b2s_cdiv((long long)batch * num_anchors, kThreads), kThreads, 0, stream>>>(
            map, batch, ny, nx, reinterpret_cast<const int4 *>(anchor_boxes), num_anchors, threshold, mask_out);
        B2S_LAUNCH_OK();
    }
    return 0;
}
