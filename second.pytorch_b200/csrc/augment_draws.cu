// augment_draws.cu -- the random numbers of prep_pointcloud's augmentation (second/data/preprocess.py:255-294) drawn on
// the device, in the layout b2s_augment reads: noise_per_object_v3_'s loc_noises / rot_noises (second/core/
// preprocess.py:582-678), random_flip's two choices (:749-769), global_rotation_v2's and global_scaling_v2's uniforms
// (:772-799), global_translate_'s normals (:885-899) and preprocess.py's np.random.shuffle(points).
// The reference draws them from numpy's global stream; here every value is a pure function of (seed, step, frame,
// stream, index) through Philox4x64-10 (the block function of numpy.random.Philox), so a frame's draws do not depend
// on how the frames are split over calls or ranks.  The contract (INTEGRATION.md, training):
//   key (seed, step), counter (frame, stream, index, 0); u(w) = (w >> 11) 2^-53; uniform lo + (hi - lo) u;
//   normals by Box-Muller from two words, r = sqrt(-2 ln(1 - u(wa))), t = 2 pi u(wb), (r cos t, r sin t);
//   stream 0: loc_noise of box b, try t at index 100 b + t; stream 1: rot_noise there; stream 2: the frame scalars
//   (index 0) and the translation (index 1); stream 3: the Feistel round keys of the shuffle, counter (f, 3, r, R).
// Kernels (one thread per output row, each finds its frame by searching the device offsets):
//   k_draw_noise  one thread per (box, try): two Philox blocks, three normals and a uniform
//   k_draw_frame  one thread per frame: flips, angle, scale and translation
//   k_draw_perm   one thread per point: the keyed permutation of its frame, a 4-round Feistel network on 2k bits
//                 cycle-walked into [0, n)
//   k_draw_step   advances the device step counter, after every other kernel of the call has read it
// Arithmetic: explicit round-to-nearest intrinsics where the contract fixes the rounding; log, sin and cos are CUDA's.
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kNumTry = B2S_AUGMENT_NUM_TRY;
constexpr unsigned long long kStreamLoc = 0, kStreamRot = 1, kStreamFrame = 2, kStreamPerm = 3;
constexpr double kTwoPi = 6.283185307179586;            // fl(2 pi), as 2.0 * math.pi
constexpr int kFeistelRounds = 4;

struct Params {
    uint64_t seed;
    const uint64_t *step;      // device
    uint64_t frame_base;
    int B;
    const int *gt_off;         // [B+1]
    int G;
    const int *point_off;      // [B+1]
    int P;
    b2s_augment_draw_params s;
    int translate;
    double *loc_noise;         // [G, kNumTry, 3] or null
    double *rot_noise;         // [G, kNumTry] or null
    double *frame;             // [B, 8]
    int *perm;                 // [P] or null
};

struct Words {
    uint64_t w[4];
};

// Philox4x64-10 (Salmon et al., SC'11; Random123's philox4x64, numpy.random.Philox's block function)
__device__ __forceinline__ Words philox(uint64_t k0, uint64_t k1, uint64_t c0, uint64_t c1, uint64_t c2, uint64_t c3)
{
    constexpr uint64_t M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
    constexpr uint64_t W0 = 0x9E3779B97F4A7C15ull, W1 = 0xBB67AE8584CAA73Bull;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += W0;
            k1 += W1;
        }
        const uint64_t hi0 = __umul64hi(M0, c0), lo0 = M0 * c0;
        const uint64_t hi1 = __umul64hi(M1, c2), lo1 = M1 * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
    }
    return Words{{c0, c1, c2, c3}};
}

__device__ __forceinline__ double u01(uint64_t w) { return __dmul_rn(__ull2double_rn(w >> 11), 0x1p-53); }

__device__ __forceinline__ double uniform(const double r[2], uint64_t w)
{
    return __dadd_rn(r[0], __dmul_rn(__dsub_rn(r[1], r[0]), u01(w)));
}

__device__ __forceinline__ double bm_radius(uint64_t w)
{
    return __dsqrt_rn(__dmul_rn(-2.0, log(__dsub_rn(1.0, u01(w)))));
}

// the three normals of a block: (w0, w1) -> (n0, n1), (w2, w3) -> n2 (its cos term)
__device__ __forceinline__ void normals3(const Words &v, double n[3])
{
    double s, c;
    const double r01 = bm_radius(v.w[0]);
    sincos(__dmul_rn(kTwoPi, u01(v.w[1])), &s, &c);
    n[0] = __dmul_rn(r01, c);
    n[1] = __dmul_rn(r01, s);
    n[2] = __dmul_rn(bm_radius(v.w[2]), cos(__dmul_rn(kTwoPi, u01(v.w[3]))));
}

// the frame of packed row `row`: the last b with off[b] <= row, -1 outside [off[0], off[B]); rows of a frame whose
// range is malformed get no frame either (b2s_augment raises B2S_STATUS_BAD_INPUT for it and never reads them)
__device__ __forceinline__ int frame_of(const int *off, int B, long long row, int &begin, int &count)
{
    if (row < off[0] || row >= off[B]) return -1;
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= row) lo = mid; else hi = mid - 1;
    }
    begin = off[lo];
    count = off[lo + 1] - begin;
    return (row >= begin && row - begin < count) ? lo : -1;
}

__global__ void __launch_bounds__(kThreads) k_draw_noise(Params p)
{
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= (long long)p.G * kNumTry) return;
    const int g = (int)(i / kNumTry), t = (int)(i - (long long)g * kNumTry);
    const uint64_t step = *p.step;
    int begin = 0, count = 0;
    const int b = frame_of(p.gt_off, p.B, g, begin, count);
    double n[3] = {0.0, 0.0, 0.0}, rn = 0.0;
    if (b >= 0) {
        const uint64_t f = p.frame_base + (uint64_t)b, idx = (uint64_t)(g - begin) * kNumTry + (uint64_t)t;
        normals3(philox(p.seed, step, f, kStreamLoc, idx, 0), n);
        for (int k = 0; k < 3; ++k) n[k] = __dmul_rn(n[k], p.s.loc_std[k]);
        rn = uniform(p.s.rot_noise, philox(p.seed, step, f, kStreamRot, idx, 0).w[0]);
    }
    double *ln = p.loc_noise + i * 3;
    ln[0] = n[0];
    ln[1] = n[1];
    ln[2] = n[2];
    p.rot_noise[i] = rn;
}

__global__ void __launch_bounds__(kThreads) k_draw_frame(Params p)
{
    const int b = blockIdx.x * kThreads + threadIdx.x;
    if (b >= p.B) return;
    const uint64_t step = *p.step, f = p.frame_base + (uint64_t)b;
    const Words v = philox(p.seed, step, f, kStreamFrame, 0, 0);
    double *fr = p.frame + (size_t)b * 8;
    fr[0] = (p.s.random_flip_y && u01(v.w[1]) < 0.5) ? 1.0 : 0.0;
    fr[1] = (p.s.random_flip_x && u01(v.w[0]) < 0.5) ? 1.0 : 0.0;
    fr[2] = p.translate ? 1.0 : 0.0;
    fr[3] = uniform(p.s.rotation, v.w[2]);
    fr[4] = uniform(p.s.scaling, v.w[3]);
    double t[3] = {0.0, 0.0, 0.0};
    if (p.translate) {
        normals3(philox(p.seed, step, f, kStreamFrame, 1, 0), t);
        t[0] = __dmul_rn(t[0], p.s.translate_std[0]);
        t[1] = __dmul_rn(t[1], p.s.translate_std[1]);
        t[2] = __dmul_rn(t[2], p.s.translate_std[0]);       // global_translate_ draws z with std[0] (:885-899)
    }
    fr[5] = t[0];
    fr[6] = t[1];
    fr[7] = t[2];
}

__global__ void __launch_bounds__(kThreads) k_draw_perm(Params p)
{
    const long long k = (long long)blockIdx.x * kThreads + threadIdx.x;     // P may be up to 2^31 - 1
    if (k >= p.P) return;
    const uint64_t step = *p.step;
    int begin = 0, n = 0;
    const int b = frame_of(p.point_off, p.B, k, begin, n);
    uint64_t x = b >= 0 ? (uint64_t)(k - begin) : 0;
    if (b >= 0 && n > 1) {
        int bits = 1;                                      // the smallest k >= 1 with 4^k >= n
        while ((1ull << (2 * bits)) < (uint64_t)n) ++bits;
        const uint64_t mask = (1ull << bits) - 1ull, f = p.frame_base + (uint64_t)b;
        do {
            uint64_t L = x >> bits, R = x & mask;
#pragma unroll
            for (int r = 0; r < kFeistelRounds; ++r) {
                const uint64_t t = L ^ (philox(p.seed, step, f, kStreamPerm, (uint64_t)r, R).w[0] & mask);
                L = R;
                R = t;
            }
            x = (L << bits) | R;
        } while (x >= (uint64_t)n);
    }
    p.perm[k] = (int)x;
}

__global__ void k_draw_step(uint64_t *step) { *step += 1; }

}  // namespace

extern "C" int b2s_augment_draws(uint64_t seed, uint64_t *step_dev, uint64_t frame_base, int batch,
                                 const int *gt_offsets, int num_gt, const int *point_offsets, int num_points,
                                 const b2s_augment_draw_params *params_host, double *loc_noise, double *rot_noise,
                                 double *frame_params, int *perm, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && batch <= 65535, "b2s_augment_draws: batch must be in [1, 65535]");
    B2S_REQUIRE(num_gt >= 0 && num_points >= 0, "b2s_augment_draws: num_gt and num_points must be >= 0");
    B2S_REQUIRE(step_dev && gt_offsets && point_offsets && params_host && frame_params,
                "b2s_augment_draws: step_dev, offsets, params_host and frame_params required");
    B2S_REQUIRE(!params_host->object_noise || num_gt == 0 || (loc_noise && rot_noise),
                "b2s_augment_draws: object noise needs loc_noise and rot_noise");
    B2S_REQUIRE(frame_base <= ~0ull - (uint64_t)batch, "b2s_augment_draws: frame_base + batch overflows 64 bits");
    Params p;
    p.seed = seed;
    p.step = step_dev;
    p.frame_base = frame_base;
    p.B = batch;
    p.gt_off = gt_offsets;
    p.G = num_gt;
    p.point_off = point_offsets;
    p.P = num_points;
    p.s = *params_host;
    p.translate = 0;
    for (int k = 0; k < 3; ++k) p.translate |= p.s.translate_std[k] != 0.0;
    p.loc_noise = loc_noise;
    p.rot_noise = rot_noise;
    p.frame = frame_params;
    p.perm = perm;
    const long long pairs = (long long)num_gt * kNumTry;
    if (p.s.object_noise && pairs > 0) {
        k_draw_noise<<<(unsigned)((pairs + kThreads - 1) / kThreads), kThreads, 0, stream>>>(p);
        B2S_LAUNCH_OK();
    }
    k_draw_frame<<<(batch + kThreads - 1) / kThreads, kThreads, 0, stream>>>(p);
    B2S_LAUNCH_OK();
    if (perm && num_points > 0) {
        k_draw_perm<<<(unsigned)(((long long)num_points + kThreads - 1) / kThreads), kThreads, 0, stream>>>(p);
        B2S_LAUNCH_OK();
    }
    k_draw_step<<<1, 1, 0, stream>>>(step_dev);
    B2S_LAUNCH_OK();
    return 0;
}
