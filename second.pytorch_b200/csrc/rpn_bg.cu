// rpn_bg.cu -- background planning for the dense RPN: b2s_rpn_strip_plan (8 x R strips), b2s_rpn_block_plan (8 x 8),
// b2s_rpn_bg_plan (16 x 16).
//
// The BEV map that enters the RPN is mostly empty: 6-8 % of the 200 x 176 pixels of a synthetic KITTI cloud hold
// data (real clouds: the camera-FOV wedge).  The output of layer l of a chain of 3x3 stride-1 pad-1 layers at pixel p
// depends on the BEV only inside the (2l+1)^2 window around p; where that window holds no data, the output is what the
// layer produces for an EMPTY frame at p -- a field that depends on the weights only (constant in the interior,
// different within l pixels of the image border, where the zero padding is felt).  The engine computes that
// empty-frame response once per layer with the very kernel that runs the layer (so the values are bit-identical to
// what the kernel would have produced) and keeps it as one halo-padded frame [H+2, W+2, C] of hi/lo planes.
// Per step, the data mask is dilated by one pixel per layer (one tiny kernel per layer); an output strip of
// k_conv3x3_tc2 (8 pixels wide, R rows high; S = 8 / R strips make one consumer warpgroup's 64-pixel accumulator tile)
// without a masked pixel is not computed -- the conv kernel's fill warps copy it from the empty-frame response -- and
// the conv kernel walks the compacted list of the remaining strips, so the work stays balanced over the SMs.  The
// engine plans 8 x 4 strips: the conv kernel's time follows the bytes it streams from L2, and 8 x 4 moves the fewest
// (finer strips compute fewer pixels but load taller windows per output row).
// Everything the reference computes is still produced; only the recomputation of a known field is skipped.
// Nor does every background strip need the field: layer l + 1 reads layer l only inside the windows of the strips it
// computes, which reach one pixel into each neighbouring strip.  b2s_rpn_strip_bands lists, per layer, the background
// strips next to a strip of the following layer (the "band"); the others are read by nothing and are left stale.  The
// last layer's band is the part of its background inside the fused tail's computed tiles, and the tail writes the
// records of its background tiles from the empty frame's records (rpn_tail.cu).
#include "common.cuh"

namespace {

constexpr int REGION = 16;        // pixels per edge of the square handled by one CTA (one thread per pixel)
constexpr int MAX_FLAGS = 32;     // granules per region: (16 / tile_h) x (16 / tile_w), tile_h >= 1, tile_w >= 8
constexpr int COMPACT_PER_THREAD = 4;

// one block per (frame, 16 x 16 region): out(p) = OR of `in` over the 3x3 window of p (outside the image: 0);
// flag of each tile_h x tile_w granule of the region (both divide 16) = OR of out over the granule's in-image pixels
__global__ void __launch_bounds__(REGION * REGION)
k_bg_layer(const uint8_t *__restrict__ in, int H, int W, int tile_h, int tile_w, int regions_h, int regions_w,
           int tiles_h, int tiles_w, uint8_t *__restrict__ out, int *__restrict__ tile_flag)
{
    const int region = blockIdx.x;
    const int rw = region % regions_w, rh = (region / regions_w) % regions_h, b = region / (regions_w * regions_h);
    const int r = threadIdx.x >> 4, c = threadIdx.x & 15;
    const int h = rh * REGION + r, w = rw * REGION + c;
    const int per_h = REGION / tile_h, per_w = REGION / tile_w;
    __shared__ int s_any[MAX_FLAGS];
    if (threadIdx.x < MAX_FLAGS) s_any[threadIdx.x] = 0;
    __syncthreads();
    if (h < H && w < W) {
        const uint8_t *f = in + (size_t)b * H * W;
        int v = 0;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int y = h + dy, x = w + dx;
                v |= (y < 0 || y >= H || x < 0 || x >= W) ? 0 : (int)f[(size_t)y * W + x];
            }
        out[((size_t)b * H + h) * W + w] = (uint8_t)(v != 0);
        if (v) s_any[(r / tile_h) * per_w + c / tile_w] = 1;
    }
    __syncthreads();
    if ((int)threadIdx.x < per_h * per_w) {
        const int th = rh * per_h + (int)threadIdx.x / per_w, tw = rw * per_w + (int)threadIdx.x % per_w;
        if (th < tiles_h && tw < tiles_w) tile_flag[((size_t)b * tiles_h + th) * tiles_w + tw] = s_any[threadIdx.x];
    }
}

// stable compaction of the ids 0 .. n-1 by flag_of(i) into list (flag 1, ascending) and, when rest is not NULL, rest
// (flag 0); each of the 1024 threads takes COMPACT_PER_THREAD consecutive ids per pass.  Returns the listed count.
template <class Flag>
__device__ int compact_ids(Flag flag_of, int n, int *list, int *rest)
{
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024 * COMPACT_PER_THREAD) {
        const int i0 = base + (int)threadIdx.x * COMPACT_PER_THREAD;
        int f[COMPACT_PER_THREAD], k1 = 0;
#pragma unroll
        for (int k = 0; k < COMPACT_PER_THREAD; ++k) {
            f[k] = i0 + k < n ? flag_of(i0 + k) : 0;
            k1 += f[k];
        }
        int total;
        const int ex = b2s_block_exscan(k1, &total);
        int wpos = s_carry + ex;                      // listed ids before i0
#pragma unroll
        for (int k = 0; k < COMPACT_PER_THREAD; ++k) {
            const int i = i0 + k;
            if (i >= n) break;
            if (f[k]) list[wpos++] = i;
            else if (rest) rest[i - wpos] = i;        // unlisted ids before i: i - (#listed ids before i)
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry += total;
        __syncthreads();
    }
    return s_carry;
}

// one block per layer: the tile ids into work (flag 1) and background (flag 0) lists
__global__ void __launch_bounds__(1024)
k_bg_compact(const int *__restrict__ tile_flag, int num_tiles, int *work_list, int *bg_list, int *counts)
{
    const int layer = blockIdx.x;
    const int *flag = tile_flag + (size_t)layer * num_tiles;
    const int n_work = compact_ids([&](int i) { return flag[i]; }, num_tiles, work_list + (size_t)layer * num_tiles,
                                   bg_list + (size_t)layer * num_tiles);
    if (threadIdx.x == 0) {
        counts[2 * layer] = n_work;
        counts[2 * layer + 1] = num_tiles - n_work;
    }
}

// blocks 0 .. num_layers - 2: the band of layer l = the strips layer l does not compute whose 3 x 3 strip
// neighbourhood in the same frame (the strip itself included) holds a strip layer l + 1 computes.
// Block num_layers - 1: the band of the last layer, read by the fused RPN tail in tiles of 8 rows x 16 columns
// (per = 8 / rows strip rows x 2 strip columns): the strips the last layer does not compute inside a computed tail tile,
// i.e. one with a computed strip.  Block num_layers: the tail's work (computed) and background tile lists.
__global__ void __launch_bounds__(1024)
k_strip_bands(const int *__restrict__ strip_flags, int num_layers, int strips_h, int strips_w, int num_strips,
              int per, int tiles_h, int tiles_w, int *band_lists, int *band_counts, int *tail_work, int *tail_bg,
              int *tail_counts)
{
    const int layer = blockIdx.x;
    const int *last = strip_flags + (size_t)(num_layers - 1) * num_strips;
    const auto tile_computed = [&](int b, int th, int tw) {
        int any = 0;
        for (int y = th * per; y < min(th * per + per, strips_h); ++y)
            for (int x = 2 * tw; x < min(2 * tw + 2, strips_w); ++x) any |= last[((size_t)b * strips_h + y) * strips_w + x];
        return any;
    };
    if (layer == num_layers) {
        const int num_tiles = num_strips / (strips_h * strips_w) * tiles_h * tiles_w;
        const int n = compact_ids([&](int i) { return tile_computed(i / (tiles_h * tiles_w), (i / tiles_w) % tiles_h,
                                                                    i % tiles_w); },
                                  num_tiles, tail_work, tail_bg);
        if (threadIdx.x == 0) {
            tail_counts[0] = n;
            tail_counts[1] = num_tiles - n;
        }
        return;
    }
    const int *cur = strip_flags + (size_t)layer * num_strips, *next = cur + num_strips;
    const auto in_band = [&](int i) {
        if (cur[i]) return 0;
        const int sw = i % strips_w, sh = (i / strips_w) % strips_h, f0 = i - sh * strips_w - sw;
        if (layer == num_layers - 1) return tile_computed(i / (strips_h * strips_w), sh / per, sw / 2);
        int any = 0;
        for (int y = max(sh - 1, 0); y <= min(sh + 1, strips_h - 1); ++y)
            for (int x = max(sw - 1, 0); x <= min(sw + 1, strips_w - 1); ++x) any |= next[f0 + y * strips_w + x];
        return any;
    };
    const int n = compact_ids(in_band, num_strips, band_lists + (size_t)layer * num_strips, nullptr);
    if (threadIdx.x == 0) band_counts[layer] = n;
}

int bg_plan(const uint8_t *occupancy, int batch, int H, int W, int num_layers, int tile_h, int tile_w,
            uint8_t *scratch, int *tile_flags, int *work_lists, int *bg_lists, int *counts, cudaStream_t stream)
{
    B2S_REQUIRE(batch >= 1 && H >= 1 && W >= 1 && num_layers >= 1 && num_layers <= 32,
                "b2s_rpn_strip_plan / b2s_rpn_block_plan / b2s_rpn_bg_plan: bad sizes");
    const int regions_h = b2s_cdiv(H, REGION), regions_w = b2s_cdiv(W, REGION);
    const int tiles_h = b2s_cdiv(H, tile_h), tiles_w = b2s_cdiv(W, tile_w);
    const int num_tiles = batch * tiles_h * tiles_w;
    const size_t map = (size_t)batch * H * W;
    const uint8_t *in = occupancy;
    for (int l = 0; l < num_layers; ++l) {
        uint8_t *out = scratch + (size_t)(l & 1) * map;
        k_bg_layer<<<batch * regions_h * regions_w, REGION * REGION, 0, stream>>>(
            in, H, W, tile_h, tile_w, regions_h, regions_w, tiles_h, tiles_w, out, tile_flags + (size_t)l * num_tiles);
        B2S_LAUNCH_OK();
        in = out;
    }
    k_bg_compact<<<num_layers, 1024, 0, stream>>>(tile_flags, num_tiles, work_lists, bg_lists, counts);
    B2S_LAUNCH_OK();
    return 0;
}

}  // namespace

extern "C" int b2s_rpn_bg_plan(const uint8_t *occupancy, int batch, int H, int W, int num_layers, uint8_t *scratch,
                               int *tile_flags, int *work_lists, int *bg_lists, int *counts, void *stream)
{
    return bg_plan(occupancy, batch, H, W, num_layers, 16, 16, scratch, tile_flags, work_lists, bg_lists, counts,
                   (cudaStream_t)stream);
}

extern "C" int b2s_rpn_block_plan(const uint8_t *occupancy, int batch, int H, int W, int num_layers, uint8_t *scratch,
                                  int *block_flags, int *work_lists, int *bg_lists, int *counts, void *stream)
{
    return bg_plan(occupancy, batch, H, W, num_layers, 8, 8, scratch, block_flags, work_lists, bg_lists, counts,
                   (cudaStream_t)stream);
}

extern "C" int b2s_rpn_strip_plan(const uint8_t *occupancy, int batch, int H, int W, int num_layers, int rows,
                                  uint8_t *scratch, int *strip_flags, int *work_lists, int *bg_lists, int *counts,
                                  void *stream)
{
    B2S_REQUIRE(rows == 1 || rows == 2 || rows == 4 || rows == 8, "b2s_rpn_strip_plan: rows must be 1, 2, 4 or 8");
    return bg_plan(occupancy, batch, H, W, num_layers, rows, 8, scratch, strip_flags, work_lists, bg_lists, counts,
                   (cudaStream_t)stream);
}

extern "C" int b2s_rpn_strip_bands(const int *strip_flags, int batch, int H, int W, int num_layers, int rows,
                                   int *band_lists, int *band_counts, int *tail_work, int *tail_bg, int *tail_counts,
                                   void *stream)
{
    B2S_REQUIRE(batch >= 1 && H >= 1 && W >= 1 && num_layers >= 1 && num_layers <= 32,
                "b2s_rpn_strip_bands: bad sizes (num_layers 1..32)");
    B2S_REQUIRE(rows == 1 || rows == 2 || rows == 4 || rows == 8, "b2s_rpn_strip_bands: rows must be 1, 2, 4 or 8");
    const int strips_h = b2s_cdiv(H, rows), strips_w = b2s_cdiv(W, 8);
    k_strip_bands<<<num_layers + 1, 1024, 0, (cudaStream_t)stream>>>(
        strip_flags, num_layers, strips_h, strips_w, batch * strips_h * strips_w, 8 / rows, b2s_cdiv(H, 8),
        b2s_cdiv(W, 16), band_lists, band_counts, tail_work, tail_bg, tail_counts);
    B2S_LAUNCH_OK();
    return 0;
}
