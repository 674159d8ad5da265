// voxelize.cu -- deterministic parallel restatement of spconv's sequential first-come voxeliser
// (b2s_voxelize, see include/b2second.h).  HBM-bound integer/byte work: every pass is a coalesced
// sweep over the point array plus hash-grid atomics.
//
// Sequential semantics reproduced bit-exactly (SURVEY.md App. A):
//   voxel id   = order of first appearance of the cell in the (frame-major) point stream
//   kept points= the first T points of the cell, in input order
//   coordinate = floor((p - lo) / vs) in fp32 with a TRUE division
//   cap        = cells first seen after max_voxels cells exist are dropped; later points of
//                already-existing cells are still added
// Parallel scheme:
//   K1 insert   : cell key -> hash slot, atomicMin(first point index)
//   K2 scan     : flag[i] = (i is the first point of its cell); exclusive scan = global first-come rank
//   K3 assign   : rank -> (frame-local id < max_voxels) -> compacted row; writes coors, hash value
//   K4 fill     : per point, count + "T smallest indices" insertion chain of atomicMin
//   K5 gather   : rows -> voxels / point_slots / fused SimpleVoxel mean
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kScanThreads = 1024;

struct VoxParams {
    float lo[3];
    float vs[3];
    int grid[3];  // x,y,z
    int key_depth;  // depth D used in the flat (b,z,y,x) hash key: the consumer's spatial shape[0] (>= grid z;
                    // SECOND's middle encoders use grid_z + 1, middle.py:139)
};

__device__ __forceinline__ int frame_of(const int *__restrict__ offsets, int batch, int i)
{
    if (offsets == nullptr) return 0;
    int lo = 0, hi = batch;  // find f with offsets[f] <= i < offsets[f+1]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (__ldg(&offsets[mid]) <= i) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void k_insert(const float *__restrict__ pts, const int *__restrict__ offsets, int P, int F,
                         int batch, VoxParams prm, unsigned long long *keys, int *first, int mask,
                         int *pslot, unsigned *status)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    // with frame offsets, offsets[batch] is the live point count (P is then only the buffer capacity)
    if (offsets != nullptr && i >= __ldg(&offsets[batch])) { pslot[i] = -1; return; }
    const float *p = pts + (size_t)i * F;
    int c[3];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        float q = __fdiv_rn(__fsub_rn(__ldg(&p[j]), prm.lo[j]), prm.vs[j]);
        float fl = floorf(q);
        if (!(fl >= 0.f && fl < (float)prm.grid[j])) ok = false;
        c[j] = (int)fl;
    }
    if (!ok) { pslot[i] = -1; return; }
    int b = frame_of(offsets, batch, i);
    unsigned long long key = b2s_flat_key(b, c[2], c[1], c[0], prm.key_depth, prm.grid[1], prm.grid[0]);
    int h = b2s_hash_insert(keys, mask, key);
    if (h < 0) { atomicOr(status, B2S_STATUS_HASH_FULL); pslot[i] = -1; return; }
    pslot[i] = h;
    atomicMin(&first[h], i);
}

// flag + per-block exclusive scan
__global__ void k_flag_scan(const int *__restrict__ pslot, const int *__restrict__ first, int P,
                            int *rank_local, int *block_sums)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int flag = 0;
    if (i < P) {
        int h = pslot[i];
        flag = (h >= 0 && first[h] == i) ? 1 : 0;
    }
    int total;
    int ex = b2s_block_exscan(flag, &total);
    if (i < P) rank_local[i] = flag ? ex : -1;
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// single block: exclusive scan of block sums (in place -> prefix, [nblk] = total), then frame bases.
__global__ void k_scan_sums_and_frames(int *block_sums, int nblk, const int *__restrict__ offsets,
                                       int P, int batch, const int *__restrict__ rank_local,
                                       const int *__restrict__ pslot, const int *__restrict__ first,
                                       int max_voxels, int *frame_rank_start /*[batch+1]*/,
                                       int *frame_row_base /*[batch+1]*/, int *num_voxels_dev,
                                       unsigned *status)
{
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblk; base += blockDim.x) {
        int idx = base + threadIdx.x;
        int v = idx < nblk ? block_sums[idx] : 0;
        int total;
        int ex = b2s_block_exscan(v, &total);
        int c = carry;
        if (idx < nblk) block_sums[idx] = c + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry = c + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) block_sums[nblk] = carry;
    __syncthreads();
    const int total_cells = carry;
    // global first-come rank at each frame start = number of first-points with index < offsets[f]
    __shared__ int s_min;
    for (int f = 0; f <= batch; ++f) {          // block-cooperative: thread t looks at point blk*1024 + t
        int off = (offsets == nullptr) ? (f == 0 ? 0 : P) : offsets[f];
        if (off >= P) {
            if (threadIdx.x == 0) frame_rank_start[f] = total_cells;
            continue;                            // `off` is block-uniform
        }
        // rank of the first "first-point" at or after `off` = smallest local rank among them in its scan block
        int blk = off / kScanThreads;
        if (threadIdx.x == 0) s_min = 0x7FFFFFFF;
        __syncthreads();
        int j = blk * kScanThreads + threadIdx.x;
        if (j >= off && j < P) {
            int rl = rank_local[j];
            if (rl >= 0) atomicMin(&s_min, rl);
        }
        __syncthreads();
        if (threadIdx.x == 0)
            frame_rank_start[f] = (s_min != 0x7FFFFFFF) ? block_sums[blk] + s_min : block_sums[blk + 1];
        __syncthreads();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int base = 0;
        for (int f = 0; f < batch; ++f) {
            int n = frame_rank_start[f + 1] - frame_rank_start[f];
            if (n > max_voxels) { atomicOr(status, B2S_STATUS_VOXEL_OVERFLOW); n = max_voxels; }
            frame_row_base[f] = base;
            num_voxels_dev[1 + f] = n;
            base += n;
        }
        frame_row_base[batch] = base;
        num_voxels_dev[0] = base;
    }
    (void)pslot; (void)first;
}

__global__ void k_assign(const int *__restrict__ pslot, const int *__restrict__ rank_local,
                         const int *__restrict__ block_prefix, const unsigned long long *__restrict__ keys,
                         int P, int batch, VoxParams prm, int max_voxels,
                         const int *__restrict__ frame_rank_start, const int *__restrict__ frame_row_base,
                         int *vals, int *coors)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int rl = rank_local[i];
    if (rl < 0) return;
    int h = pslot[i];
    int g = block_prefix[i / kScanThreads] + rl;
    unsigned long long key = keys[h];
    const unsigned long long W = prm.grid[0], H = prm.grid[1], D = prm.key_depth;
    int x = (int)(key % W);
    unsigned long long r = key / W;
    int y = (int)(r % H);
    r /= H;
    int z = (int)(r % D);
    int b = (int)(r / D);
    int local = g - frame_rank_start[b];
    if (local >= max_voxels) return;  // dropped cell: hash value stays -1
    int row = frame_row_base[b] + local;
    vals[h] = row;
    int4 c = make_int4(b, z, y, x);
    *reinterpret_cast<int4 *>(coors + (size_t)row * 4) = c;
    (void)batch;
}

__global__ void k_fill(const int *__restrict__ pslot, const int *__restrict__ vals, int P, int T,
                       int *num, int *slots)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int h = pslot[i];
    if (h < 0) return;
    int row = vals[h];
    if (row < 0) return;
    atomicAdd(&num[row], 1);
    int *s = slots + (size_t)row * T;
    // slot values only ever decrease: if the last slot already holds a smaller index, i cannot be
    // among the T smallest.
    if (*((volatile int *)&s[T - 1]) < i) return;
    int v = i;
    for (int t = 0; t < T; ++t) {
        int old = atomicMin(&s[t], v);
        if (old > v) v = old;          // we displaced `old`: carry it down the chain
        if (v == B2S_INF_IDX) break;   // displaced an empty slot: done
    }
}

// one thread per (row, t): materialise voxels and finalise point_slots
__global__ void k_gather(const float *__restrict__ pts, int F, int T, const int *__restrict__ num_total,
                         int *slots, float *voxels)
{
    long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int n = *num_total;
    if (gid >= (long long)n * T) return;
    int idx = slots[gid];
    bool valid = idx != B2S_INF_IDX;
    if (!valid) slots[gid] = -1;
    if (voxels != nullptr) {
        float *dst = voxels + gid * F;
        if (valid) {
            const float *src = pts + (size_t)idx * F;
            for (int f = 0; f < F; ++f) dst[f] = __ldg(&src[f]);
        } else {
            for (int f = 0; f < F; ++f) dst[f] = 0.f;
        }
    }
}

// one thread per row: clamp the count, fused VFE
__global__ void k_finish(const float *__restrict__ pts, int F, int T, const int *__restrict__ num_total,
                         const int *__restrict__ slots, int *num, int vfe_mode, int vfe_nf, float *vfe_out)
{
    int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= *num_total) return;
    int n = min(num[row], T);
    num[row] = n;
    if (vfe_mode == B2S_VFE_NONE) return;
    float acc[8];
#pragma unroll
    for (int f = 0; f < 8; ++f) acc[f] = 0.f;
    const int *s = slots + (size_t)row * T;
    for (int t = 0; t < n; ++t) {
        const float *src = pts + (size_t)s[t] * F;
#pragma unroll
        for (int f = 0; f < 8; ++f)
            if (f < vfe_nf) acc[f] = __fadd_rn(acc[f], __ldg(&src[f]));
    }
    float fn = (float)n;
#pragma unroll
    for (int f = 0; f < 8; ++f)
        if (f < vfe_nf) acc[f] = __fdiv_rn(acc[f], fn);
    if (vfe_mode == B2S_VFE_MEAN) {
        float *o = vfe_out + (size_t)row * vfe_nf;
#pragma unroll
        for (int f = 0; f < 8; ++f)
            if (f < vfe_nf) o[f] = acc[f];
    } else {  // MEAN_RADIUS: [norm(xy), mean[2:nf]]
        float *o = vfe_out + (size_t)row * (vfe_nf - 1);
        o[0] = sqrtf(__fadd_rn(__fmul_rn(acc[0], acc[0]), __fmul_rn(acc[1], acc[1])));
#pragma unroll
        for (int f = 2; f < 8; ++f)
            if (f < vfe_nf) o[f - 1] = acc[f];
    }
}

// SimpleVoxel / SimpleVoxelRadius over voxels that arrive already gathered ([rows, T, F], zero padded): the same
// sequential fp32 sum in slot order and true division as k_finish
__global__ void k_vfe_mean(const float *__restrict__ voxels, const int *__restrict__ num, const int *__restrict__ n_dev,
                           int cap_rows, int T, int F, int vfe_mode, int vfe_nf, float *vfe_out)
{
    const int n_rows = min(*n_dev, cap_rows);
    for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n_rows; row += gridDim.x * blockDim.x) {
        const int n = min(num[row], T);
        float acc[8];
#pragma unroll
        for (int f = 0; f < 8; ++f) acc[f] = 0.f;
        const float *v = voxels + (size_t)row * T * F;
        for (int t = 0; t < n; ++t) {
#pragma unroll
            for (int f = 0; f < 8; ++f)
                if (f < vfe_nf) acc[f] = __fadd_rn(acc[f], __ldg(&v[(size_t)t * F + f]));
        }
        const float fn = (float)n;
#pragma unroll
        for (int f = 0; f < 8; ++f)
            if (f < vfe_nf) acc[f] = __fdiv_rn(acc[f], fn);
        if (vfe_mode == B2S_VFE_MEAN) {
            float *o = vfe_out + (size_t)row * vfe_nf;
#pragma unroll
            for (int f = 0; f < 8; ++f)
                if (f < vfe_nf) o[f] = acc[f];
        } else {
            float *o = vfe_out + (size_t)row * (vfe_nf - 1);
            o[0] = sqrtf(__fadd_rn(__fmul_rn(acc[0], acc[0]), __fmul_rn(acc[1], acc[1])));
#pragma unroll
            for (int f = 2; f < 8; ++f)
                if (f < vfe_nf) o[f - 1] = acc[f];
        }
    }
}

struct VoxWorkspace {
    int *pslot, *first, *rank_local, *block_sums, *frame_rank_start, *frame_row_base;
};

size_t carve(VoxWorkspace *w, char *base, int P, int batch, int hash_cap)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += b2s_align(bytes); return base ? base + o : nullptr; };
    int nblk = b2s_cdiv(P > 0 ? P : 1, kScanThreads);
    int *pslot = (int *)take(sizeof(int) * (size_t)(P > 0 ? P : 1));
    int *first = (int *)take(sizeof(int) * (size_t)hash_cap);
    int *rank_local = (int *)take(sizeof(int) * (size_t)(P > 0 ? P : 1));
    int *block_sums = (int *)take(sizeof(int) * (size_t)(nblk + 1));
    int *frs = (int *)take(sizeof(int) * (size_t)(batch + 1));
    int *frb = (int *)take(sizeof(int) * (size_t)(batch + 1));
    if (w) { w->pslot = pslot; w->first = first; w->rank_local = rank_local; w->block_sums = block_sums;
             w->frame_rank_start = frs; w->frame_row_base = frb; }
    return off;
}

}  // namespace

extern "C" int b2s_voxelize_hash_capacity(int num_points)
{
    long long want = 2ll * (num_points > 0 ? num_points : 1);
    long long cap = 1024;
    while (cap < want) cap <<= 1;
    return (int)cap;
}

extern "C" size_t b2s_voxelize_workspace_bytes(int num_points, int batch, int max_voxels, int max_points)
{
    (void)max_voxels; (void)max_points;
    return carve(nullptr, nullptr, num_points, batch, b2s_voxelize_hash_capacity(num_points));
}

extern "C" int b2s_voxelize(const float *points, const int *frame_offsets_dev, int num_points, int num_feat,
                            int batch, const float *range_lo, const float *voxel_size, const int *grid,
                            int max_points, int max_voxels, int *coors, int *num_points_per_voxel,
                            int *point_slots, float *voxels, int vfe_mode, int vfe_num_features,
                            float *vfe_out, int *num_voxels_dev, unsigned long long *hash_keys,
                            int *hash_vals, int hash_cap, int hash_key_depth, void *workspace,
                            size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    const int P = num_points, F = num_feat, T = max_points;
    B2S_REQUIRE(hash_key_depth == 0 || hash_key_depth >= grid[2],
                "b2s_voxelize: hash_key_depth must be 0 (= grid z) or >= grid z");
    B2S_REQUIRE(P >= 0 && F >= 3 && batch >= 1 && T >= 1 && max_voxels >= 1, "b2s_voxelize: bad sizes");
    B2S_REQUIRE((hash_cap & (hash_cap - 1)) == 0 && hash_cap >= 2 * (P > 0 ? P : 1),
                "b2s_voxelize: hash_cap must be a power of two >= 2*num_points");
    B2S_REQUIRE(vfe_mode == B2S_VFE_NONE || (vfe_num_features >= 3 && vfe_num_features <= 8 &&
                vfe_num_features <= F && vfe_out != nullptr), "b2s_voxelize: bad vfe arguments");
    B2S_REQUIRE((long long)batch * grid[0] * grid[1] * grid[2] > 0, "b2s_voxelize: bad grid");
    VoxWorkspace w;
    size_t need = carve(&w, (char *)workspace, P, batch, hash_cap);
    B2S_REQUIRE(workspace_bytes >= need, "b2s_voxelize: workspace too small (%zu < %zu)", workspace_bytes, need);
    VoxParams prm;
    for (int j = 0; j < 3; ++j) { prm.lo[j] = range_lo[j]; prm.vs[j] = voxel_size[j]; prm.grid[j] = grid[j]; }
    prm.key_depth = hash_key_depth > 0 ? hash_key_depth : grid[2];
    const size_t cap_rows = (size_t)batch * max_voxels;
    B2S_CUDA_OK(cudaMemsetAsync(hash_keys, 0xFF, sizeof(unsigned long long) * (size_t)hash_cap, stream));
    B2S_CUDA_OK(cudaMemsetAsync(hash_vals, 0xFF, sizeof(int) * (size_t)hash_cap, stream));
    B2S_CUDA_OK(cudaMemsetAsync(w.first, 0x7F, sizeof(int) * (size_t)hash_cap, stream));
    B2S_CUDA_OK(cudaMemsetAsync(num_points_per_voxel, 0, sizeof(int) * cap_rows, stream));
    B2S_CUDA_OK(cudaMemsetAsync(point_slots, 0x7F, sizeof(int) * cap_rows * T, stream));
    const int nblk = b2s_cdiv(P > 0 ? P : 1, kScanThreads);
    if (P > 0) {
        k_insert<<<b2s_cdiv(P, kThreads), kThreads, 0, stream>>>(points, frame_offsets_dev, P, F, batch, prm,
                                                                 hash_keys, w.first, hash_cap - 1, w.pslot,
                                                                 status_dev);
        B2S_LAUNCH_OK();
    }
    k_flag_scan<<<nblk, kScanThreads, 0, stream>>>(w.pslot, w.first, P, w.rank_local, w.block_sums);
    B2S_LAUNCH_OK();
    k_scan_sums_and_frames<<<1, kScanThreads, 0, stream>>>(w.block_sums, nblk, frame_offsets_dev, P, batch,
                                                           w.rank_local, w.pslot, w.first, max_voxels,
                                                           w.frame_rank_start, w.frame_row_base,
                                                           num_voxels_dev, status_dev);
    B2S_LAUNCH_OK();
    if (P > 0) {
        k_assign<<<b2s_cdiv(P, kThreads), kThreads, 0, stream>>>(w.pslot, w.rank_local, w.block_sums, hash_keys,
                                                                 P, batch, prm, max_voxels, w.frame_rank_start,
                                                                 w.frame_row_base, hash_vals, coors);
        B2S_LAUNCH_OK();
        k_fill<<<b2s_cdiv(P, kThreads), kThreads, 0, stream>>>(w.pslot, hash_vals, P, T, num_points_per_voxel,
                                                               point_slots);
        B2S_LAUNCH_OK();
    }
    // rows <= min(P, cap_rows): size the grids by that bound, kernels exit on the device-side count
    const long long max_rows = (long long)((size_t)P < cap_rows ? (size_t)P : cap_rows);
    if (max_rows > 0) {
        k_gather<<<b2s_cdiv(max_rows * T, kThreads), kThreads, 0, stream>>>(points, F, T, num_voxels_dev,
                                                                            point_slots, voxels);
        B2S_LAUNCH_OK();
        k_finish<<<b2s_cdiv(max_rows, kThreads), kThreads, 0, stream>>>(points, F, T, num_voxels_dev, point_slots,
                                                                        num_points_per_voxel, vfe_mode,
                                                                        vfe_num_features, vfe_out);
        B2S_LAUNCH_OK();
    }
    return 0;
}

extern "C" int b2s_vfe_mean(const float *voxels, const int *num_points_per_voxel, const int *num_rows_dev, int cap_rows,
                            int T, int F, int vfe_mode, int vfe_num_features, float *vfe_out, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(vfe_mode == B2S_VFE_MEAN || vfe_mode == B2S_VFE_MEAN_RADIUS, "b2s_vfe_mean: vfe_mode must be 1 or 2");
    B2S_REQUIRE(T >= 1 && F >= 1 && vfe_num_features >= (vfe_mode == B2S_VFE_MEAN_RADIUS ? 2 : 1) &&
                vfe_num_features <= 8 && vfe_num_features <= F, "b2s_vfe_mean: bad feature counts");
    if (cap_rows <= 0) return 0;
    int blocks = b2s_cdiv(cap_rows, kThreads);
    if (blocks > 132 * 8) blocks = 132 * 8;
    k_vfe_mean<<<blocks, kThreads, 0, stream>>>(voxels, num_points_per_voxel, num_rows_dev, cap_rows, T, F, vfe_mode,
                                                vfe_num_features, vfe_out);
    B2S_LAUNCH_OK();
    return 0;
}
