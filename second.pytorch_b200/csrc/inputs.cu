// inputs.cu -- on-GPU input path in front of the voxelizer (SURVEY.md §8(f)1):
//   b2s_transform_sweep : one NuScenes sweep -> [x', y', z', dt] rows of the merged cloud
//                         (second/data/nuscenes_dataset.py:166-185: points[:, :3] @ R.T + t, time lag column)
//   b2s_crop_convex     : keep the points strictly inside a convex polytope given by its inward-normal planes, in
//                         input order (KITTI velodyne_reduced FOV crop: second/core/box_np_ops.py:682-693 ->
//                         second/core/geometry.py:149-172,358-395), compacted straight into a frame slot of the
//                         voxelizer's point buffer
// Both are HBM-bound streaming kernels; the arithmetic is the reference's float64 (numpy promotes the float32 points
// against float64 calibration), with explicit mul/add so no FMA contraction changes a rounding.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxPlanes = 16;

struct Rigid {
    double r[9], t[3];
};

__global__ void k_transform_sweep(const float *__restrict__ in, int P, int F_in, Rigid m, float dt, int identity,
                                  float *__restrict__ out)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
        const float *p = in + (size_t)i * F_in;
        const float x = __ldg(&p[0]), y = __ldg(&p[1]), z = __ldg(&p[2]);
        float4 o;
        if (identity) {
            o = make_float4(x, y, z, dt);
        } else {
            // row = p @ R^T: component j = p . R[j,:], float64, left to right; rounded to float32 when it is stored back
            // into the float32 sweep array; then `+= t` is float32 + float64 -> float64 -> float32 again
            float q[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                double s = __dmul_rn((double)x, m.r[3 * j]);
                s = __dadd_rn(s, __dmul_rn((double)y, m.r[3 * j + 1]));
                s = __dadd_rn(s, __dmul_rn((double)z, m.r[3 * j + 2]));
                q[j] = (float)__dadd_rn((double)(float)s, m.t[j]);
            }
            o = make_float4(q[0], q[1], q[2], dt);
        }
        *reinterpret_cast<float4 *>(out + (size_t)i * 4) = o;
    }
}

struct Planes {
    double n[kMaxPlanes][4];   // (a, b, c, d): inside <=> a x + b y + c z + d < 0 for every plane
    int count;
};

__device__ __forceinline__ bool inside(const Planes &pl, float x, float y, float z)
{
    for (int k = 0; k < pl.count; ++k) {
        double s = __dmul_rn((double)x, pl.n[k][0]);
        s = __dadd_rn(s, __dmul_rn((double)y, pl.n[k][1]));
        s = __dadd_rn(s, __dmul_rn((double)z, pl.n[k][2]));
        s = __dadd_rn(s, pl.n[k][3]);
        if (s >= 0.0) return false;
    }
    return true;
}

// pass 1: per-block count of kept points
__global__ void __launch_bounds__(kThreads)
k_crop_count(const float *__restrict__ pts, int P, int F, Planes pl, int *__restrict__ block_counts)
{
    const int i = blockIdx.x * kThreads + threadIdx.x;
    bool keep = false;
    if (i < P) {
        const float *p = pts + (size_t)i * F;
        keep = inside(pl, __ldg(&p[0]), __ldg(&p[1]), __ldg(&p[2]));
    }
    int total;
    b2s_block_exscan(keep ? 1 : 0, &total);
    if (threadIdx.x == 0) block_counts[blockIdx.x] = total;
}

// pass 2 (one block): exclusive scan of the block counts; publishes the frame's end offset
__global__ void __launch_bounds__(1024)
k_crop_scan(int *block_counts, int nblocks, int *offsets_dev, int out_cap_rows, unsigned *status)
{
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nblocks ? block_counts[i] : 0;
        int total;
        const int ex = b2s_block_exscan(v, &total);
        const int carry = s_carry;
        if (i < nblocks) block_counts[i] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const int start = offsets_dev[0];
        int end = start + s_carry;
        if (end > out_cap_rows) {               // never write past the buffer: drop the tail, raise the flag
            end = out_cap_rows;
            if (status) atomicOr(status, B2S_STATUS_ROWS_OVERFLOW);
        }
        offsets_dev[1] = end;
    }
}

// pass 3: order-preserving compaction into out[start + rank]
__global__ void __launch_bounds__(kThreads)
k_crop_emit(const float *__restrict__ pts, int P, int F, Planes pl, const int *__restrict__ block_offsets,
            const int *__restrict__ offsets_dev, int out_cap_rows, float *__restrict__ out)
{
    const int i = blockIdx.x * kThreads + threadIdx.x;
    bool keep = false;
    const float *p = pts + (size_t)i * F;
    if (i < P) keep = inside(pl, __ldg(&p[0]), __ldg(&p[1]), __ldg(&p[2]));
    int total;
    const int ex = b2s_block_exscan(keep ? 1 : 0, &total);
    if (!keep) return;
    const int row = offsets_dev[0] + block_offsets[blockIdx.x] + ex;
    if (row >= out_cap_rows) return;
    float *o = out + (size_t)row * F;
    for (int f = 0; f < F; ++f) o[f] = __ldg(&p[f]);
}

}  // namespace

extern "C" int b2s_transform_sweep(const float *points_in, int num_points, int feat_in, const double *rotation_host,
                                   const double *translation_host, float time_lag, float *out, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(num_points >= 0 && feat_in >= 3, "b2s_transform_sweep: points must have at least x, y, z");
    B2S_REQUIRE(((uintptr_t)out & 15) == 0, "b2s_transform_sweep: out must be 16-byte aligned");
    if (num_points == 0) return 0;
    Rigid m;
    const int identity = rotation_host == nullptr;
    for (int i = 0; i < 9; ++i) m.r[i] = identity ? (i % 4 == 0 ? 1.0 : 0.0) : rotation_host[i];
    for (int i = 0; i < 3; ++i) m.t[i] = (identity || !translation_host) ? 0.0 : translation_host[i];
    int blocks = b2s_cdiv(num_points, kThreads);
    if (blocks > 132 * 8) blocks = 132 * 8;
    k_transform_sweep<<<blocks, kThreads, 0, stream>>>(points_in, num_points, feat_in, m, time_lag, identity, out);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" size_t b2s_crop_workspace_bytes(int num_points)
{
    return sizeof(int) * (size_t)(b2s_cdiv(num_points > 0 ? num_points : 1, kThreads) + 1);
}

extern "C" int b2s_crop_convex(const float *points, int num_points, int num_feat, const double *planes_host,
                               int num_planes, float *out_points, int out_cap_rows, int *offsets_dev, void *workspace,
                               size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(num_points >= 0 && num_feat >= 3 && num_planes >= 1 && num_planes <= kMaxPlanes,
                "b2s_crop_convex: 1..16 planes, points with at least x, y, z");
    B2S_REQUIRE(workspace_bytes >= b2s_crop_workspace_bytes(num_points), "b2s_crop_convex: workspace too small");
    Planes pl;
    pl.count = num_planes;
    for (int k = 0; k < num_planes; ++k)
        for (int j = 0; j < 4; ++j) pl.n[k][j] = planes_host[4 * k + j];
    int *block_counts = (int *)workspace;
    const int nblocks = b2s_cdiv(num_points > 0 ? num_points : 1, kThreads);
    k_crop_count<<<nblocks, kThreads, 0, stream>>>(points, num_points, num_feat, pl, block_counts);
    B2S_LAUNCH_OK();
    k_crop_scan<<<1, 1024, 0, stream>>>(block_counts, nblocks, offsets_dev, out_cap_rows, status_dev);
    B2S_LAUNCH_OK();
    k_crop_emit<<<nblocks, kThreads, 0, stream>>>(points, num_points, num_feat, pl, block_counts, offsets_dev, out_cap_rows,
                                                  out_points);
    B2S_LAUNCH_OK();
    return 0;
}
