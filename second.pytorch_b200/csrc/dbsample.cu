// dbsample.cu -- ground-truth database sampling of prep_pointcloud (second/data/preprocess.py:210-249) for a batch of
// frames: DataBaseSamplerV2.sample_all / sample_class_v2 (second/core/sample_ops.py:95-285) after the host has drawn
// the candidates (b2second.dbsample.draw), then the point removal and the concatenation.
//
// Acceptance rule.  sample_class_v2 builds the all-pairs BEV collision matrix of [avoid_coll_boxes; candidates of one
// class] (box_collision_test on center_to_corner_box2d corners), clears the diagonal and walks the candidates in order:
// a candidate whose row still holds a collision is rejected and its row and column are cleared.  So candidate i is
// rejected exactly when its BEV box collides with any of
//   - a ground truth of the frame (every row of gt_boxes, whatever its class mask);
//   - an accepted candidate of an earlier class (only accepted boxes join avoid_coll_boxes);
//   - an accepted earlier candidate of its own class (a rejected one's column was cleared);
//   - any later candidate of its own class, accepted later or not (its column is still set when row i is read).
// Candidates of later classes play no part.  Accepted boxes keep the order class, then candidate order.
//
// Kernels (after memsets of points_out and the candidates' and points' ranks):
//   k_db_frame<T>   one CTA per frame: the frame's and its candidates' BEV corners and standup boxes in shared memory;
//                   for each candidate in order every other box is tested in parallel and one block vote decides.
//                   Writes each candidate's rank among the frame's accepted ones, its first output point and the 3-D
//                   planes of its box, and the frame's counts.
//   k_db_rank<T>    one CTA per frame: with remove_points a point inside an accepted box is dropped (points_in_rbbox:
//                   origin-0.5 box, points_in_convex_polygon_3d_jit); stable rank of the kept points.
//   k_db_offsets    the packed point and box offsets of the output.
//   k_db_boxes<T>   one thread per output box row: the frame's boxes, then its accepted boxes.
//   k_db_points<T>  one thread per input point and per candidate point: the accepted objects' points translated by
//                   their box centre (s_points[:, :3] += box[:3], in the box dtype, stored as float32), then the
//                   frame's kept points in their original order.
// Bad inputs.  A frame's range in point_offsets, gt_offsets or cand_offsets is used only when it lies inside the array
// and after every earlier entry and before every later one, so the ranges in use never overlap; a range that fails
// raises B2S_STATUS_BAD_INPUT and that part of the frame is empty.  A candidate whose object id is outside the database
// or whose cand_point_offsets step differs from the object's point count is rejected (B2S_STATUS_BAD_INPUT).  No write
// goes past the output capacity: totals that would exceed it raise B2S_STATUS_BAD_INPUT and are clamped.
// The box geometry is box_geom.cuh's, shared with augment.cu.
#include "box_geom.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxBoxes = B2S_DBSAMPLE_MAX_BOXES;

struct Params {
    const float *points;            // [P, F]
    const int *point_off;           // [B+1]
    int P, F, B;
    const void *boxes;              // [G, ndim] of T
    const int *gt_off;              // [B+1]
    const uint8_t *valid;           // [G]
    const int *classes;             // [G]
    const float *importance;        // [G] or null (ones)
    int G, ndim;
    const int *cand_obj;            // [C] database object ids
    const int *cand_group;          // [C] sample-group index
    const int *cand_off;            // [B+1]
    const int *cand_pt_off;         // [C+1] prefix of the candidates' point counts
    int C, CP;
    const float *db_points;         // [NP, F]
    const long long *db_point_off;  // [N+1]
    const void *db_boxes;           // [N, ndim] of T
    const int *db_class;            // [N] 1-based class of each object
    int N;
    float sample_importance;
    int remove_points;
    // workspace
    void *planes;                   // [C, 24] of T
    int *acc_rank;                  // [C] rank among the frame's accepted candidates, -1 rejected
    int *acc_pt;                    // [C] first output point of an accepted candidate, relative to the frame
    int *acc_cand;                  // [C] candidate row of the frame's r-th accepted one, at cand_off[b] + r
    int *cand_frame;                // [C] frame of a candidate in a valid range
    int *kept_rank;                 // [P] rank among the frame's kept points, -1 dropped or in no valid range
    int *pt_frame;                  // [P] frame of a kept point
    int *frame_ngt, *frame_nacc, *frame_nspts, *frame_nkeep;   // [B]
    int *frame_c0, *frame_nc;       // [B] the frame's candidate range in use (empty when invalid)
    // outputs
    float *points_out;              // [P + CP, F]
    int *point_off_out;             // [B+1]
    void *boxes_out;                // [G + C, ndim]
    int *gt_off_out;                // [B+1]
    uint8_t *valid_out;             // [G + C]
    int *classes_out;               // [G + C]
    float *importance_out;          // [G + C]
    int *src_object;                // [G + C] database object of a sampled row, -1 for the frame's own
    uint8_t *accepted;              // [C]
    unsigned *status;
};

// the last b in [0, B) with off[b] <= k (off nondecreasing over the searched entries)
__device__ __forceinline__ int frame_of(const int *off, int B, int k)
{
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= k) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// the CTA's frame range [off[b], off[b+1]) of an array of n rows, usable when it is ordered, inside [0, n], not before
// any earlier entry and not after any later one (so the usable ranges of a batch are disjoint); every thread gets the
// same answer.  Unusable: f0 = f1 = 0.
__device__ __noinline__ bool block_frame_range(const int *off, int B, int b, int n, int &f0, int &f1)
{
    f0 = off[b];
    f1 = off[b + 1];
    bool ok = f0 >= 0 && f1 >= f0 && f1 <= n;
    for (int j = threadIdx.x; j <= B && ok; j += blockDim.x) {
        const int v = off[j];
        if ((j < b && v > f0) || (j > b + 1 && v < f1)) ok = false;
    }
    ok = __syncthreads_and(ok ? 1 : 0) != 0;
    if (!ok) f0 = f1 = 0;
    return ok;
}

__device__ __forceinline__ int obj_points(const Params &p, int obj)
{
    return (int)(p.db_point_off[obj + 1] - p.db_point_off[obj]);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_db_frame(Params p)
{
    extern __shared__ __align__(16) unsigned char smem[];
    T *s_cor = reinterpret_cast<T *>(smem);                 // [kMaxBoxes][8]
    T *s_su = s_cor + (size_t)kMaxBoxes * 8;                // [kMaxBoxes][4]
    uint8_t *s_acc = reinterpret_cast<uint8_t *>(s_su + (size_t)kMaxBoxes * 4);   // [kMaxBoxes]
    uint8_t *s_bad = s_acc + kMaxBoxes;                     // [kMaxBoxes]
    const int b = blockIdx.x, tid = threadIdx.x;
    int f0, f1, c0, c1;
    const bool gt_ok = block_frame_range(p.gt_off, p.B, b, p.G, f0, f1);      // bad: no ground truth
    const bool cand_ok = block_frame_range(p.cand_off, p.B, b, p.C, c0, c1);  // bad: no candidates
    if (tid == 0 && (!gt_ok || !cand_ok)) atomicOr(p.status, B2S_STATUS_BAD_INPUT);
    const int ng = f1 - f0, nc = c1 - c0, n = ng + nc;
    const bool capped = n > kMaxBoxes;
    if (capped && tid == 0) atomicOr(p.status, B2S_STATUS_DB_BOX_CAP);
    const T *boxes = static_cast<const T *>(p.boxes);
    const T *db_boxes = static_cast<const T *>(p.db_boxes);

    if (!capped) {
        for (int i = tid; i < n; i += kThreads) {
            const T *bx;
            if (i < ng) {
                bx = boxes + (size_t)(f0 + i) * p.ndim;
            } else {
                const int k = i - ng, obj = p.cand_obj[c0 + k];
                const bool bad = obj < 0 || obj >= p.N ||
                                 p.cand_pt_off[c0 + k + 1] - p.cand_pt_off[c0 + k] != obj_points(p, obj);
                s_bad[k] = bad;
                s_acc[k] = 0;
                if (bad) {
                    atomicOr(p.status, B2S_STATUS_BAD_INPUT);
                    continue;
                }
                bx = db_boxes + (size_t)obj * p.ndim;
                box_planes<T>(bx, static_cast<T *>(p.planes) + (size_t)(c0 + k) * 24);
            }
            T c[8], su[4];
            corners2d<T>(bx[0], bx[1], bx[3], bx[4], bx[6], c);
            standup<T>(c, su);
#pragma unroll
            for (int k = 0; k < 8; ++k) s_cor[i * 8 + k] = c[k];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_su[i * 4 + k] = su[k];
        }
        __syncthreads();
        for (int k = 0; k < nc; ++k) {
            const int i = ng + k;
            const int grp = p.cand_group[c0 + k];
            bool hit = false;
            if (!s_bad[k]) {
                for (int j = tid; j < n && !hit; j += kThreads) {
                    if (j == i) continue;
                    bool against = j < ng;                          // a ground truth of the frame
                    if (!against) {
                        const int kj = j - ng;
                        against = kj < k ? s_acc[kj] != 0                      // accepted earlier candidate
                                         : (!s_bad[kj] && p.cand_group[c0 + kj] == grp);   // later one of its class
                    }
                    if (against && collide<T>(s_cor + i * 8, s_su + i * 4, s_cor + j * 8, s_su + j * 4)) hit = true;
                }
            }
            const int any = __syncthreads_or(hit ? 1 : 0);
            if (tid == 0) s_acc[k] = !any && !s_bad[k];
            __syncthreads();
        }
    }
    if (tid == 0) {
        int r = 0, pts = 0;
        for (int k = 0; k < nc; ++k) {
            const bool acc = !capped && s_acc[k];
            p.cand_frame[c0 + k] = b;
            p.accepted[c0 + k] = acc;
            p.acc_rank[c0 + k] = acc ? r : -1;
            if (acc) {
                p.acc_pt[c0 + k] = pts;
                p.acc_cand[c0 + r] = c0 + k;
                pts += obj_points(p, p.cand_obj[c0 + k]);
                ++r;
            }
        }
        p.frame_ngt[b] = ng;
        p.frame_nacc[b] = r;
        p.frame_nspts[b] = pts;
        p.frame_c0[b] = c0;
        p.frame_nc[b] = nc;
    }
}

// remove_points_after_sample: a point inside any accepted box of its frame is dropped; then the stable rank of the
// frame's kept points, a block ballot per chunk on top of the earlier chunks' count
template <typename T>
__global__ void __launch_bounds__(kThreads) k_db_rank(Params p)
{
    __shared__ int s_warp[kThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    int q0, q1;
    if (!block_frame_range(p.point_off, p.B, b, p.P, q0, q1) && tid == 0) atomicOr(p.status, B2S_STATUS_BAD_INPUT);
    const int c0 = p.frame_c0[b], c1 = c0 + p.frame_nc[b];
    const T *planes = static_cast<const T *>(p.planes);
    int kept_before = 0;
    for (int k0 = q0; k0 < q1; k0 += kThreads) {
        const int k = k0 + tid;
        bool kept = k < q1;
        if (kept && p.remove_points) {
            const float *in = p.points + (size_t)k * p.F;
            const float x = in[0], y = in[1], z = in[2];
            for (int c = c0; c < c1 && kept; ++c)
                if (p.acc_rank[c] >= 0 && in_planes<T>(planes + (size_t)c * 24, x, y, z)) kept = false;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, kept);
        if ((tid & 31) == 0) s_warp[tid >> 5] = __popc(bal);
        __syncthreads();
        int total = 0, before = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
            if (w < (tid >> 5)) before += s_warp[w];
            total += s_warp[w];
        }
        if (kept) {
            p.kept_rank[k] = kept_before + before + __popc(bal & ((1u << (tid & 31)) - 1u));
            p.pt_frame[k] = b;
        }
        kept_before += total;
        __syncthreads();                                   // s_warp is reused by the next chunk
    }
    if (tid == 0) p.frame_nkeep[b] = kept_before;
}

// output offsets: per frame its sampled points then its kept points, its boxes then its accepted boxes (B is small)
__global__ void k_db_offsets(Params p)
{
    if (threadIdx.x != 0) return;
    // with usable (disjoint) ranges the totals fit; only inconsistent cand_point_offsets can push the points past it
    const long long pcap = (long long)p.P + p.CP, gcap = (long long)p.G + p.C;
    long long pr = 0, gr = 0;
    for (int b = 0; b < p.B; ++b) {
        p.point_off_out[b] = (int)min(pr, pcap);
        p.gt_off_out[b] = (int)min(gr, gcap);
        pr += p.frame_nspts[b] + p.frame_nkeep[b];
        gr += p.frame_ngt[b] + p.frame_nacc[b];
    }
    const bool over = pr > pcap || gr > gcap;
    p.point_off_out[p.B] = (int)min(pr, pcap);
    p.gt_off_out[p.B] = (int)min(gr, gcap);
    if (over) atomicOr(p.status, B2S_STATUS_BAD_INPUT);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_db_boxes(Params p)
{
    const int o = blockIdx.x * kThreads + threadIdx.x;
    if (o >= p.G + p.C) return;
    T *dst = static_cast<T *>(p.boxes_out) + (size_t)o * p.ndim;
    if (o >= p.gt_off_out[p.B]) {                           // rows past the packed boxes: zeros, source -1
        for (int k = 0; k < p.ndim; ++k) dst[k] = T(0);
        p.valid_out[o] = 0;
        p.classes_out[o] = 0;
        p.importance_out[o] = 0.f;
        p.src_object[o] = -1;
        return;
    }
    const int b = frame_of(p.gt_off_out, p.B, o);
    const int r = o - p.gt_off_out[b], ng = p.frame_ngt[b];
    if (r < ng) {
        const int g = p.gt_off[b] + r;
        const T *src = static_cast<const T *>(p.boxes) + (size_t)g * p.ndim;
        for (int k = 0; k < p.ndim; ++k) dst[k] = src[k];
        p.valid_out[o] = p.valid[g];
        p.classes_out[o] = p.classes[g];
        p.importance_out[o] = p.importance ? p.importance[g] : 1.f;
        p.src_object[o] = -1;
    } else {
        const int obj = p.cand_obj[p.acc_cand[p.frame_c0[b] + (r - ng)]];
        const T *src = static_cast<const T *>(p.db_boxes) + (size_t)obj * p.ndim;
        for (int k = 0; k < p.ndim; ++k) dst[k] = src[k];
        p.valid_out[o] = 1;
        p.classes_out[o] = p.db_class[obj];
        p.importance_out[o] = p.sample_importance;
        p.src_object[o] = obj;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_db_points(Params p)
{
    const int t = blockIdx.x * kThreads + threadIdx.x;
    const long long cap = (long long)p.P + p.CP;
    if (t < p.P) {                                          // a frame's own point
        const int r = p.kept_rank[t];
        if (r < 0) return;
        const int b = p.pt_frame[t];
        const long long row = (long long)p.point_off_out[b] + p.frame_nspts[b] + r;
        if (row >= min(cap, (long long)p.point_off_out[b + 1])) return;
        const float *in = p.points + (size_t)t * p.F;
        float *out = p.points_out + (size_t)row * p.F;
        for (int c = 0; c < p.F; ++c) out[c] = in[c];
        return;
    }
    const int u = t - p.P;                                  // a candidate's point
    if (u >= p.CP) return;
    const int k = frame_of(p.cand_pt_off, p.C, u);
    if (p.acc_rank[k] < 0) return;                          // rejected, or outside every usable candidate range
    const int obj = p.cand_obj[k], local = u - p.cand_pt_off[k];
    if (local < 0 || local >= obj_points(p, obj)) return;
    const int b = p.cand_frame[k];
    const long long row = (long long)p.point_off_out[b] + p.acc_pt[k] + local;
    if (row >= min(cap, (long long)p.point_off_out[b + 1])) return;
    const float *in = p.db_points + (size_t)(p.db_point_off[obj] + local) * p.F;
    const T *bx = static_cast<const T *>(p.db_boxes) + (size_t)obj * p.ndim;
    float *out = p.points_out + (size_t)row * p.F;
    out[0] = pt_add(in[0], bx[0]);
    out[1] = pt_add(in[1], bx[1]);
    out[2] = pt_add(in[2], bx[2]);
    for (int c = 3; c < p.F; ++c) out[c] = in[c];
}

struct Ws {
    void *planes;
    int *acc_rank, *acc_pt, *acc_cand, *cand_frame, *kept_rank, *pt_frame, *frame;
    size_t bytes;
};

Ws carve(void *base, int batch, int num_points, int num_cand)
{
    Ws w;
    char *p = (char *)base;
    size_t off = 0;
    const size_t c = (size_t)(num_cand > 0 ? num_cand : 1), np_ = (size_t)(num_points > 0 ? num_points : 1);
    w.planes = p + off;
    off += b2s_align(sizeof(double) * 24 * c);
    w.acc_rank = (int *)(p + off);
    off += b2s_align(sizeof(int) * c);
    w.acc_pt = (int *)(p + off);
    off += b2s_align(sizeof(int) * c);
    w.acc_cand = (int *)(p + off);
    off += b2s_align(sizeof(int) * c);
    w.cand_frame = (int *)(p + off);
    off += b2s_align(sizeof(int) * c);
    w.kept_rank = (int *)(p + off);
    off += b2s_align(sizeof(int) * np_);
    w.pt_frame = (int *)(p + off);
    off += b2s_align(sizeof(int) * np_);
    w.frame = (int *)(p + off);
    off += b2s_align(sizeof(int) * 6 * (size_t)batch);
    w.bytes = off;
    return w;
}

template <typename T>
size_t frame_smem() { return sizeof(T) * (size_t)kMaxBoxes * 12 + 2 * (size_t)kMaxBoxes; }

template <typename T>
int launch(Params p, cudaStream_t stream)
{
    const size_t smem = frame_smem<T>();
    static bool attr_done[64] = {false};
    int dev = 0;
    B2S_CUDA_OK(cudaGetDevice(&dev));
    if (!attr_done[dev & 63]) {
        B2S_CUDA_OK(cudaFuncSetAttribute(k_db_frame<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[dev & 63] = true;
    }
    const size_t rows = (size_t)p.P + (size_t)p.CP;
    if (rows) B2S_CUDA_OK(cudaMemsetAsync(p.points_out, 0, sizeof(float) * rows * (size_t)p.F, stream));
    if (p.C > 0) {                          // candidates outside every valid frame range: rejected
        B2S_CUDA_OK(cudaMemsetAsync(p.acc_rank, 0xFF, sizeof(int) * (size_t)p.C, stream));
        B2S_CUDA_OK(cudaMemsetAsync(p.accepted, 0, (size_t)p.C, stream));
    }
    if (p.P > 0)                            // points outside every usable frame range: dropped
        B2S_CUDA_OK(cudaMemsetAsync(p.kept_rank, 0xFF, sizeof(int) * (size_t)p.P, stream));
    k_db_frame<T><<<p.B, kThreads, smem, stream>>>(p);
    B2S_LAUNCH_OK();
    k_db_rank<T><<<p.B, kThreads, 0, stream>>>(p);
    B2S_LAUNCH_OK();
    k_db_offsets<<<1, 32, 0, stream>>>(p);
    B2S_LAUNCH_OK();
    if (p.G + p.C > 0) {
        k_db_boxes<T><<<(p.G + p.C + kThreads - 1) / kThreads, kThreads, 0, stream>>>(p);
        B2S_LAUNCH_OK();
    }
    if (rows) {
        k_db_points<T><<<(unsigned)((rows + kThreads - 1) / kThreads), kThreads, 0, stream>>>(p);
        B2S_LAUNCH_OK();
    }
    return 0;
}

}  // namespace

extern "C" size_t b2s_db_sample_workspace_bytes(int batch, int num_points, int num_cand)
{
    if (batch <= 0 || num_points < 0 || num_cand < 0) return 0;
    return carve(nullptr, batch, num_points, num_cand).bytes;
}

extern "C" int b2s_db_sample(const float *points, int num_points, int num_feat, const int *point_offsets, int batch,
                             const void *gt_boxes, int gt_double, int box_ndim, int num_gt, const int *gt_offsets,
                             const uint8_t *gt_valid, const int *gt_classes, const float *gt_importance,
                             const int *cand_obj, const int *cand_group, const int *cand_offsets,
                             const int *cand_point_offsets, int num_cand, int num_cand_points, const float *db_points,
                             const long long *db_point_offsets, const void *db_boxes, const int *db_classes,
                             int num_objects, float sample_importance, int remove_points, float *points_out,
                             int *point_offsets_out, void *boxes_out, int *gt_offsets_out, uint8_t *valid_out,
                             int *classes_out, float *importance_out, int *src_object, uint8_t *accepted,
                             void *workspace, size_t workspace_bytes, unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && batch <= 65535, "b2s_db_sample: batch must be in [1, 65535]");
    B2S_REQUIRE(num_points >= 0 && num_feat >= 3, "b2s_db_sample: num_points must be >= 0 and num_feat >= 3");
    B2S_REQUIRE(num_gt >= 0 && (box_ndim == 7 || box_ndim == 9), "b2s_db_sample: num_gt must be >= 0 and box_ndim 7 or 9");
    B2S_REQUIRE(gt_double == 0 || gt_double == 1, "b2s_db_sample: gt_double must be 0 or 1");
    B2S_REQUIRE(remove_points == 0 || remove_points == 1, "b2s_db_sample: remove_points must be 0 or 1");
    B2S_REQUIRE(num_cand >= 0 && num_cand_points >= 0 && num_objects >= 0, "b2s_db_sample: negative candidate or "
                "object count");
    B2S_REQUIRE((size_t)num_points + (size_t)num_cand_points <= (size_t)0x7fffffff && (size_t)num_gt + num_cand <=
                (size_t)0x7fffffff, "b2s_db_sample: output rows must fit in int32");
    B2S_REQUIRE(point_offsets && gt_offsets && cand_offsets && cand_point_offsets, "b2s_db_sample: offsets required");
    B2S_REQUIRE(num_cand > 0 || num_cand_points == 0, "b2s_db_sample: candidate points without candidates");
    B2S_REQUIRE(num_points == 0 || points, "b2s_db_sample: points required");
    B2S_REQUIRE(num_gt == 0 || (gt_boxes && gt_valid && gt_classes), "b2s_db_sample: gt inputs required");
    B2S_REQUIRE(num_cand == 0 || (cand_obj && cand_group && db_point_offsets && db_boxes && db_classes &&
                                  num_objects > 0), "b2s_db_sample: candidates need the database");
    B2S_REQUIRE(num_cand_points == 0 || db_points, "b2s_db_sample: db_points required");
    B2S_REQUIRE((num_points + num_cand_points == 0 || points_out) && point_offsets_out && gt_offsets_out &&
                (num_gt + num_cand == 0 || (boxes_out && valid_out && classes_out && importance_out && src_object)) &&
                (num_cand == 0 || accepted) && status_dev, "b2s_db_sample: outputs required");
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= b2s_db_sample_workspace_bytes(batch, num_points, num_cand),
                "b2s_db_sample: workspace too small");
    const Ws w = carve(workspace, batch, num_points, num_cand);
    Params p;
    p.points = points;
    p.point_off = point_offsets;
    p.P = num_points;
    p.F = num_feat;
    p.B = batch;
    p.boxes = gt_boxes;
    p.gt_off = gt_offsets;
    p.valid = gt_valid;
    p.classes = gt_classes;
    p.importance = gt_importance;
    p.G = num_gt;
    p.ndim = box_ndim;
    p.cand_obj = cand_obj;
    p.cand_group = cand_group;
    p.cand_off = cand_offsets;
    p.cand_pt_off = cand_point_offsets;
    p.C = num_cand;
    p.CP = num_cand_points;
    p.db_points = db_points;
    p.db_point_off = db_point_offsets;
    p.db_boxes = db_boxes;
    p.db_class = db_classes;
    p.N = num_objects;
    p.sample_importance = sample_importance;
    p.remove_points = remove_points;
    p.planes = w.planes;
    p.acc_rank = w.acc_rank;
    p.acc_pt = w.acc_pt;
    p.acc_cand = w.acc_cand;
    p.cand_frame = w.cand_frame;
    p.kept_rank = w.kept_rank;
    p.pt_frame = w.pt_frame;
    p.frame_ngt = w.frame;
    p.frame_nacc = w.frame + batch;
    p.frame_nspts = w.frame + 2 * (size_t)batch;
    p.frame_nkeep = w.frame + 3 * (size_t)batch;
    p.frame_c0 = w.frame + 4 * (size_t)batch;
    p.frame_nc = w.frame + 5 * (size_t)batch;
    p.points_out = points_out;
    p.point_off_out = point_offsets_out;
    p.boxes_out = boxes_out;
    p.gt_off_out = gt_offsets_out;
    p.valid_out = valid_out;
    p.classes_out = classes_out;
    p.importance_out = importance_out;
    p.src_object = src_object;
    p.accepted = accepted;
    p.status = status_dev;
    return gt_double ? launch<double>(p, stream) : launch<float>(p, stream);
}
