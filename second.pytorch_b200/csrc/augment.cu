// augment.cu -- the augmentation of prep_pointcloud (second/data/preprocess.py:255-294) after ground-truth database
// sampling, for a batch of frames:
//   noise_per_object_v3_ with num_try tries and no per-object global rotation (second/core/preprocess.py:582-678):
//     noise_per_box (:244-273) with box_collision_test (:803-883), points_transform_ (:450-466), box3d_transform_
//     (:469-475); the point test points_in_convex_polygon_3d_jit (second/core/geometry.py:149-229) on
//     center_to_corner_box3d(origin = [0.5, 0.5, 0.5]) surfaces (box_np_ops.py:377-402, :764-782, geometry.py:332-355);
//   random_flip (:749-769), global_rotation_v2 (:781-799), global_scaling_v2 (:772-778), global_translate_ (:885-899);
//   filter_gt_box_outside_range_by_center (:153-164), limit_period(0.5, 2 pi) and np.random.shuffle(points).
// Kernels:
//   k_aug_frame<T>   one CTA per frame.  Box planes for the point test; then pose selection: frame corners and standup
//                    boxes in shared memory, for each valid box in order the (try, other box) pairs of kChunk tries are
//                    tested in parallel and the smallest collision-free try wins (the reference's first j), its corners
//                    replace the box's before the next box starts.  Then every box's transformed values, its kept flag
//                    and its rank among the frame's kept boxes.
//   k_aug_pack<T>    every CTA scans the per-frame kept counts and scatters its boxes to the packed output.
//   k_aug_points<T>  one thread per output point: source row perm[k], first valid box whose pre-noise 3-D box holds it,
//                    that box's transform, then the global ops.
// Arithmetic follows the reference's dtypes and step order: points float32, boxes T (float32 KITTI, float64 NuScenes),
// random draws float64.  Every step is an explicit round-to-nearest intrinsic so --fmad=true cannot contract it.
// The box geometry (corners, collision test, planes, point test) is box_geom.cuh's, shared with dbsample.cu.
#include "box_geom.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kChunk = 32;                 // tries evaluated together; one warp ballot picks the first free one
constexpr int kMaxBoxes = B2S_AUGMENT_MAX_BOXES;
constexpr int kSelNone = -1;               // no collision-free try: the box moves by zero
constexpr int kSelSkipped = -2;            // frame over kMaxBoxes: no object noise in that frame

struct Params {
    const float *points;        // [P, F]
    const int *point_off;       // [B+1]
    int P, F, B;
    const void *boxes;          // [G, ndim] of T
    const int *gt_off;          // [B+1]
    const uint8_t *valid;       // [G]
    const int *classes;         // [G]
    const float *importance;    // [G] or null (ones)
    int G, ndim;
    const double *loc_noise;    // [G, num_try, 3]
    const double *rot_noise;    // [G, num_try]
    int num_try, object_noise;
    const double *frame;        // [B, 8]: flip_y, flip_x, translate, angle, scale, tx, ty, tz
    const int *perm;            // [P] frame-local source rows, or null
    float range[4];             // x0, y0, x1, y1 (float32, point_cloud_range[[0, 1, 3, 4]])
    // workspace
    void *planes;               // [G, 6, 4] of T: inward normal (3) and d
    void *tboxes;               // [G, ndim] of T: transformed boxes
    int *rank;                  // [G]: rank among the frame's kept boxes, -1 dropped
    int *frame_kept;            // [B]
    // outputs
    float *points_out;          // [P, F]
    int *point_box;             // [P] or null
    void *boxes_out;            // [G, ndim]
    int *gt_off_out;            // [B+1]
    int *classes_out, *src_out; // [G]
    float *importance_out;      // [G]
    int *selected;              // [G]
    unsigned *status;
};

__device__ __forceinline__ bool frame_range(const int *off, int b, int n, int &f0, int &f1)
{
    f0 = off[b];
    f1 = off[b + 1];
    return f0 >= 0 && f1 >= f0 && f1 <= n;
}


// points_in_convex_polygon_jit of one point against the clockwise range rectangle minmax_to_corner_2d builds
template <typename T>
__device__ __forceinline__ bool in_range(const float r[4], T px, T py)
{
    using M = Ar<T>;
    const float dx = __fsub_rn(r[2], r[0]), dy = __fsub_rn(r[3], r[1]);
    const float poly[8] = {r[0], r[1], r[0], __fadd_rn(r[1], dy), __fadd_rn(r[0], dx), __fadd_rn(r[1], dy),
                           __fadd_rn(r[0], dx), r[1]};
    for (int k = 0; k < 4; ++k) {
        const int kp = (k + 3) & 3;
        const float v0 = __fsub_rn(poly[2 * k], poly[2 * kp]), v1 = __fsub_rn(poly[2 * k + 1], poly[2 * kp + 1]);
        T cross = M::mul(T(v1), M::sub(T(poly[2 * k]), px));
        cross = M::sub(cross, M::mul(T(v0), M::sub(T(poly[2 * k + 1]), py)));
        if (cross >= T(0)) return false;
    }
    return true;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_aug_frame(Params p)
{
    using M = Ar<T>;
    extern __shared__ __align__(16) unsigned char smem[];
    T *s_cor = reinterpret_cast<T *>(smem);                 // [kMaxBoxes][8]
    T *s_su = s_cor + (size_t)kMaxBoxes * 8;                // [kMaxBoxes][4]
    T *s_try = s_su + (size_t)kMaxBoxes * 4;                // [kChunk][8]
    T *s_trysu = s_try + kChunk * 8;                        // [kChunk][4]
    __shared__ unsigned s_coll;
    __shared__ int s_warp[kThreads / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    int f0, f1, q0, q1;
    const bool gt_ok = frame_range(p.gt_off, b, p.G, f0, f1);
    const bool pt_ok = frame_range(p.point_off, b, p.P, q0, q1);
    if (tid == 0 && (!gt_ok || !pt_ok)) atomicOr(p.status, B2S_STATUS_BAD_INPUT);
    if (!gt_ok) f0 = f1 = 0;                                // the frame is treated as having no ground truth
    const int n = f1 - f0;
    const T *boxes = static_cast<const T *>(p.boxes);
    const bool noise = p.object_noise && n > 0 && n <= kMaxBoxes;
    if (p.object_noise && n > kMaxBoxes && tid == 0) atomicOr(p.status, B2S_STATUS_AUG_BOX_CAP);

    if (noise) {
        T *planes = static_cast<T *>(p.planes);
        for (int i = tid; i < n; i += kThreads) {
            const T *bx = boxes + (size_t)(f0 + i) * p.ndim;
            box_planes<T>(bx, planes + (size_t)(f0 + i) * 24);
            T c[8], su[4];
            corners2d<T>(bx[0], bx[1], bx[3], bx[4], bx[6], c);
            standup<T>(c, su);
#pragma unroll
            for (int k = 0; k < 8; ++k) s_cor[i * 8 + k] = c[k];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_su[i * 4 + k] = su[k];
        }
        __syncthreads();
        for (int i = 0; i < n; ++i) {
            const int g = f0 + i;
            if (!p.valid[g]) {
                if (tid == 0) p.selected[g] = kSelNone;
                continue;
            }
            const T *bx = boxes + (size_t)g * p.ndim;
            const T bx0 = bx[0], bx1 = bx[1];
            int sel = kSelNone;
            for (int j0 = 0; j0 < p.num_try; j0 += kChunk) {
                const int nt = min(kChunk, p.num_try - j0);
                if (tid < nt) {
                    const int j = j0 + tid;
                    const double rn = p.rot_noise[(size_t)g * p.num_try + j];
                    const double *ln = p.loc_noise + ((size_t)g * p.num_try + j) * 3;
                    const T c = M::from(cos(rn)), s = M::from(sin(rn));
                    const double ox = __dadd_rn((double)bx0, ln[0]), oy = __dadd_rn((double)bx1, ln[1]);
                    T cc[8], su[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        T x = M::sub(s_cor[i * 8 + 2 * k], bx0), y = M::sub(s_cor[i * 8 + 2 * k + 1], bx1);
                        rot2<T>(x, y, c, s);
                        cc[2 * k] = add_f64<T>(x, ox);
                        cc[2 * k + 1] = add_f64<T>(y, oy);
                    }
                    standup<T>(cc, su);
#pragma unroll
                    for (int k = 0; k < 8; ++k) s_try[tid * 8 + k] = cc[k];
#pragma unroll
                    for (int k = 0; k < 4; ++k) s_trysu[tid * 4 + k] = su[k];
                }
                if (tid == 0) s_coll = nt < 32 ? ~0u << nt : 0u;    // tries past num_try count as colliding
                __syncthreads();
                for (int w = tid; w < nt * n; w += kThreads) {
                    const int jj = w / n, k = w - jj * n;
                    if (k == i || ((*(volatile unsigned *)&s_coll >> jj) & 1u)) continue;
                    if (collide<T>(s_try + jj * 8, s_trysu + jj * 4, s_cor + k * 8, s_su + k * 4))
                        atomicOr(&s_coll, 1u << jj);
                }
                __syncthreads();
                const unsigned free_ = ~s_coll;
                if (free_ != 0u) {
                    const int jj = __ffs(free_) - 1;
                    sel = j0 + jj;
                    if (tid < 8) s_cor[i * 8 + tid] = s_try[jj * 8 + tid];
                    if (tid < 4) s_su[i * 4 + tid] = s_trysu[jj * 4 + tid];
                }
                __syncthreads();
                if (sel >= 0) break;
            }
            if (tid == 0) p.selected[g] = sel;
        }
    } else {
        for (int i = tid; i < n; i += kThreads) p.selected[f0 + i] = p.object_noise ? kSelSkipped : kSelNone;
    }
    __syncthreads();

    // boxes: box3d_transform_, then the global ops, the range filter and limit_period
    const double *fr = p.frame + (size_t)b * 8;
    const bool flip_y = fr[0] != 0.0, flip_x = fr[1] != 0.0, translate = fr[2] != 0.0;
    const double angle = fr[3], scale = fr[4];
    T *tb = static_cast<T *>(p.tboxes);
    int kept_before = 0;
    for (int c0 = 0; c0 < n; c0 += kThreads) {
        const int i = c0 + tid;
        bool kept = false;
        if (i < n) {
            const int g = f0 + i;
            const T *bx = boxes + (size_t)g * p.ndim;
            T v[9];
            for (int k = 0; k < p.ndim && k < 9; ++k) v[k] = bx[k];
            if (p.valid[g]) {
                const int sel = p.selected[g];
                if (p.object_noise && sel != kSelSkipped) {
                    const double *ln = sel >= 0 ? p.loc_noise + ((size_t)g * p.num_try + sel) * 3 : nullptr;
                    const double rn = sel >= 0 ? p.rot_noise[(size_t)g * p.num_try + sel] : 0.0;
                    for (int k = 0; k < 3; ++k) v[k] = add_f64<T>(v[k], ln ? ln[k] : 0.0);
                    v[6] = add_f64<T>(v[6], rn);
                }
                const bool vel = p.ndim == 9;
                if (flip_y) {
                    v[1] = -v[1];
                    v[6] = M::add(-v[6], M::from(M_PI));
                    if (vel) v[8] = -v[8];
                }
                if (flip_x) {
                    v[0] = -v[0];
                    v[6] = -v[6];
                    if (vel) v[7] = -v[7];
                }
                {
                    const T c = M::from(cos(angle)), s = M::from(sin(angle));
                    rot2<T>(v[0], v[1], c, s);
                    v[6] = M::add(v[6], M::from(angle));
                    if (vel) {                                    // float64 boxes @ a float32 matrix
                        const T c32 = T(__double2float_rn(cos(angle))), s32 = T(__double2float_rn(sin(angle)));
                        rot2<T>(v[7], v[8], c32, s32);
                    }
                }
                const T sc = M::from(scale);
                for (int k = 0; k < 6; ++k) v[k] = M::mul(v[k], sc);
                if (vel) {
                    v[7] = M::mul(v[7], sc);
                    v[8] = M::mul(v[8], sc);
                }
                if (translate)
                    for (int k = 0; k < 3; ++k) v[k] = add_f64<T>(v[k], fr[5 + k]);
                kept = in_range<T>(p.range, v[0], v[1]);
                if (kept) {
                    const T period = M::from(2.0 * M_PI);
                    v[6] = M::sub(v[6], M::mul(floor(M::add(M::div(v[6], period), T(0.5))), period));
                    T *o = tb + (size_t)g * p.ndim;
                    for (int k = 0; k < p.ndim; ++k) o[k] = k < 9 ? v[k] : bx[k];
                }
            }
        }
        // stable rank among the frame's kept boxes: a block ballot per chunk on top of the earlier chunks' count
        const unsigned bal = __ballot_sync(0xffffffffu, kept);
        if ((tid & 31) == 0) s_warp[tid >> 5] = __popc(bal);
        __syncthreads();
        int total = 0, before = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
            if (w < (tid >> 5)) before += s_warp[w];
            total += s_warp[w];
        }
        if (i < n) p.rank[f0 + i] = kept ? kept_before + before + __popc(bal & ((1u << (tid & 31)) - 1u)) : -1;
        kept_before += total;
        __syncthreads();                                   // s_warp is reused by the next chunk
    }
    if (tid == 0) p.frame_kept[b] = kept_before;
}

// exclusive scan of the per-frame kept counts (every CTA, B is small) and the scatter of its range of boxes
template <typename T>
__global__ void __launch_bounds__(kThreads) k_aug_pack(Params p)
{
    __shared__ int s_part[kThreads];
    __shared__ int s_total;
    const int tid = threadIdx.x;
    // frame_start[b] = sum of frame_kept[< b]; each thread sums a contiguous run of frames
    const int per = (p.B + kThreads - 1) / kThreads;
    int acc = 0;
    for (int b = tid * per; b < min(p.B, (tid + 1) * per); ++b) acc += p.frame_kept[b];
    s_part[tid] = acc;
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int t = 0; t < kThreads; ++t) {
            const int v = s_part[t];
            s_part[t] = run;
            run += v;
        }
        s_total = run;
    }
    __syncthreads();
    if (blockIdx.x == 0) {
        int run = s_part[tid];
        for (int b = tid * per; b < min(p.B, (tid + 1) * per); ++b) {
            p.gt_off_out[b] = run;
            run += p.frame_kept[b];
        }
        if (tid == kThreads - 1) p.gt_off_out[p.B] = run;
    }
    const int g = blockIdx.x * kThreads + tid;
    if (g >= p.G) return;
    if (g >= s_total) {                                     // rows past the kept boxes: zeros, source row -1
        T *dst = static_cast<T *>(p.boxes_out) + (size_t)g * p.ndim;
        for (int k = 0; k < p.ndim; ++k) dst[k] = T(0);
        p.classes_out[g] = 0;
        p.importance_out[g] = 0.f;
        p.src_out[g] = -1;
    }
    const int r = p.rank[g];
    if (r < 0) return;
    // the frame of box g: the last b with gt_off[b] <= g among frames with valid offsets
    int lo = 0, hi = p.B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (p.gt_off[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const int b = lo;
    int start = s_part[b / per];
    for (int bb = (b / per) * per; bb < b; ++bb) start += p.frame_kept[bb];
    const int o = start + r;
    if (o >= p.G) return;                                   // only reachable with bad gt_offsets (status raised)
    const T *src = static_cast<const T *>(p.tboxes) + (size_t)g * p.ndim;
    T *dst = static_cast<T *>(p.boxes_out) + (size_t)o * p.ndim;
    for (int k = 0; k < p.ndim; ++k) dst[k] = src[k];
    p.classes_out[o] = p.classes[g];
    p.importance_out[o] = p.importance ? p.importance[g] : 1.f;
    p.src_out[o] = g;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_aug_points(Params p)
{
    const int k = blockIdx.x * kThreads + threadIdx.x;
    if (k >= p.P) return;
    // frame of output row k: the last b with point_off[b] <= k (rows past point_off[B] pass through unchanged)
    int b = -1;
    if (k >= p.point_off[0] && k < p.point_off[p.B]) {
        int lo = 0, hi = p.B - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (p.point_off[mid] <= k) lo = mid; else hi = mid - 1;
        }
        b = lo;
    }
    int src = k, q0 = 0, q1 = 0;
    bool ok = b >= 0 && frame_range(p.point_off, b, p.P, q0, q1) && k < q1;
    if (ok && p.perm) {
        const int m = p.perm[k];
        if (m >= 0 && m < q1 - q0) {
            src = q0 + m;
        } else {
            atomicOr(p.status, B2S_STATUS_BAD_INPUT);
        }
    }
    const float *in = p.points + (size_t)src * p.F;
    float x = in[0], y = in[1], z = in[2];
    int moved_by = -1;
    if (ok && p.object_noise) {
        int f0, f1;
        if (frame_range(p.gt_off, b, p.G, f0, f1)) {
            const T *planes = static_cast<const T *>(p.planes);
            const T *boxes = static_cast<const T *>(p.boxes);
            for (int g = f0; g < f1; ++g) {
                if (!p.valid[g]) continue;
                if (!in_planes<T>(planes + (size_t)g * 24, x, y, z)) continue;
                const int sel = p.selected[g];
                if (sel == kSelSkipped) break;
                moved_by = g;
                const T *bx = boxes + (size_t)g * p.ndim;
                const double rn = sel >= 0 ? p.rot_noise[(size_t)g * p.num_try + sel] : 0.0;
                const double *ln = sel >= 0 ? p.loc_noise + ((size_t)g * p.num_try + sel) * 3 : nullptr;
                const float c = __double2float_rn(cos(rn)), s = __double2float_rn(sin(rn));
                x = pt_sub(x, bx[0]);
                y = pt_sub(y, bx[1]);
                z = pt_sub(z, bx[2]);
                rot2<float>(x, y, c, s);
                x = pt_add(x, bx[0]);
                y = pt_add(y, bx[1]);
                z = pt_add(z, bx[2]);
                x = pt_add(x, ln ? ln[0] : 0.0);
                y = pt_add(y, ln ? ln[1] : 0.0);
                z = pt_add(z, ln ? ln[2] : 0.0);
                break;
            }
        }
    }
    if (ok) {
        const double *fr = p.frame + (size_t)b * 8;
        if (fr[0] != 0.0) y = -y;
        if (fr[1] != 0.0) x = -x;
        const double angle = fr[3];
        rot2<float>(x, y, __double2float_rn(cos(angle)), __double2float_rn(sin(angle)));
        const float sc = __double2float_rn(fr[4]);
        x = __fmul_rn(x, sc);
        y = __fmul_rn(y, sc);
        z = __fmul_rn(z, sc);
        if (fr[2] != 0.0) {
            x = pt_add(x, fr[5]);
            y = pt_add(y, fr[6]);
            z = pt_add(z, fr[7]);
        }
    }
    float *out = p.points_out + (size_t)k * p.F;
    out[0] = x;
    out[1] = y;
    out[2] = z;
    for (int c = 3; c < p.F; ++c) out[c] = in[c];
    if (p.point_box) p.point_box[k] = moved_by;
}

struct Ws {
    void *planes, *tboxes;
    int *rank, *frame_kept;
    size_t bytes;
};

Ws carve(void *base, int batch, int num_gt, int box_ndim)
{
    Ws w;
    char *p = (char *)base;
    size_t off = 0;
    const size_t g = (size_t)(num_gt > 0 ? num_gt : 1);
    w.planes = p + off;
    off += b2s_align(sizeof(double) * 24 * g);
    w.tboxes = p + off;
    off += b2s_align(sizeof(double) * (size_t)box_ndim * g);
    w.rank = (int *)(p + off);
    off += b2s_align(sizeof(int) * g);
    w.frame_kept = (int *)(p + off);
    off += b2s_align(sizeof(int) * (size_t)batch);
    w.bytes = off;
    return w;
}

template <typename T>
size_t frame_smem() { return sizeof(T) * ((size_t)kMaxBoxes * 12 + kChunk * 12); }

template <typename T>
int launch(const Params &p, cudaStream_t stream)
{
    const size_t smem = frame_smem<T>();
    static bool attr_done[64] = {false};
    int dev = 0;
    B2S_CUDA_OK(cudaGetDevice(&dev));
    if (!attr_done[dev & 63]) {
        B2S_CUDA_OK(cudaFuncSetAttribute(k_aug_frame<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_done[dev & 63] = true;
    }
    if (p.G > 0) B2S_CUDA_OK(cudaMemsetAsync(p.rank, 0xFF, sizeof(int) * (size_t)p.G, stream));   // -1: not kept
    k_aug_frame<T><<<p.B, kThreads, smem, stream>>>(p);
    B2S_LAUNCH_OK();
    k_aug_pack<T><<<max(1, (p.G + kThreads - 1) / kThreads), kThreads, 0, stream>>>(p);
    B2S_LAUNCH_OK();
    if (p.P > 0) {
        k_aug_points<T><<<(p.P + kThreads - 1) / kThreads, kThreads, 0, stream>>>(p);
        B2S_LAUNCH_OK();
    }
    return 0;
}

}  // namespace

extern "C" size_t b2s_augment_workspace_bytes(int batch, int num_gt, int box_ndim)
{
    if (batch <= 0 || num_gt < 0 || box_ndim <= 0) return 0;
    return carve(nullptr, batch, num_gt, box_ndim).bytes;
}

extern "C" int b2s_augment(const float *points, int num_points, int num_feat, const int *point_offsets, int batch,
                           const void *gt_boxes, int gt_double, int box_ndim, int num_gt, const int *gt_offsets,
                           const uint8_t *gt_valid, const int *gt_classes, const float *gt_importance,
                           const double *loc_noise, const double *rot_noise, int num_try, int object_noise,
                           const double *frame_params, const int *perm, const float *range_host, float *points_out,
                           int *point_box, void *boxes_out, int *gt_offsets_out, int *classes_out,
                           float *importance_out, int *src_out, int *selected, void *workspace, size_t workspace_bytes,
                           unsigned *status_dev, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && batch <= 65535, "b2s_augment: batch must be in [1, 65535]");
    B2S_REQUIRE(num_points >= 0 && num_feat >= 3, "b2s_augment: num_points must be >= 0 and num_feat >= 3");
    B2S_REQUIRE(num_gt >= 0 && (box_ndim == 7 || box_ndim == 9), "b2s_augment: num_gt must be >= 0 and box_ndim 7 or 9");
    B2S_REQUIRE(gt_double == 0 || gt_double == 1, "b2s_augment: gt_double must be 0 or 1");
    B2S_REQUIRE(object_noise == 0 || object_noise == 1, "b2s_augment: object_noise must be 0 or 1");
    B2S_REQUIRE(!object_noise || num_gt == 0 || (loc_noise && rot_noise && num_try >= 1),
                "b2s_augment: object noise needs loc_noise, rot_noise and num_try >= 1");
    B2S_REQUIRE(point_offsets && gt_offsets && frame_params && range_host, "b2s_augment: offsets, frame_params and "
                "range required");
    B2S_REQUIRE(num_points == 0 || (points && points_out), "b2s_augment: points and points_out required");
    B2S_REQUIRE(num_gt == 0 || (gt_boxes && gt_valid && gt_classes && boxes_out && classes_out && importance_out &&
                                src_out && selected),
                "b2s_augment: gt inputs and outputs required");
    B2S_REQUIRE(gt_offsets_out && status_dev, "b2s_augment: gt_offsets_out and status_dev required");
    B2S_REQUIRE(workspace != nullptr && workspace_bytes >= b2s_augment_workspace_bytes(batch, num_gt, box_ndim),
                "b2s_augment: workspace too small");
    const Ws w = carve(workspace, batch, num_gt, box_ndim);
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
    p.loc_noise = loc_noise;
    p.rot_noise = rot_noise;
    p.num_try = num_try;
    p.object_noise = object_noise;
    p.frame = frame_params;
    p.perm = perm;
    for (int k = 0; k < 4; ++k) p.range[k] = range_host[k];
    p.planes = w.planes;
    p.tboxes = w.tboxes;
    p.rank = w.rank;
    p.frame_kept = w.frame_kept;
    p.points_out = points_out;
    p.point_box = point_box;
    p.boxes_out = boxes_out;
    p.gt_off_out = gt_offsets_out;
    p.classes_out = classes_out;
    p.src_out = src_out;
    p.importance_out = importance_out;
    p.selected = selected;
    p.status = status_dev;
    return gt_double ? launch<double>(p, stream) : launch<float>(p, stream);
}
