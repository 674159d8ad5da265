// rpn_bg.cu -- background-tile planning for the dense RPN (b2s_rpn_bg_plan, b2s_rpn_bg_fill).
//
// The BEV map that enters the RPN is mostly empty: 6-8 % of the 200 x 176 pixels of a synthetic KITTI cloud hold
// data (real clouds: the camera-FOV wedge).  The output of layer l of a chain of 3x3 stride-1 pad-1 layers at pixel p
// depends on the BEV only inside the (2l+1)^2 window around p; where that window holds no data, the output is what the
// layer produces for an EMPTY frame at p -- a field that depends on the weights only (constant in the interior,
// different within l pixels of the image border, where the zero padding is felt).  The engine computes that
// empty-frame response once per layer with the very kernel that runs the layer (so the values are bit-identical to
// what the kernel would have produced) and keeps it as one halo-padded frame [H+2, W+2, C] of hi/lo planes.
// Per step, the data mask is dilated by one pixel per layer (one tiny kernel per layer); a 16 x 16 output tile of
// k_conv3x3_tc2 without a masked pixel is not computed -- it is copied from the empty-frame response (by the conv
// kernel's own epilogue warps, or b2s_rpn_bg_fill) -- and the conv kernel walks the compacted list of the remaining
// tiles, so the work stays balanced over the SMs.
// Everything the reference computes is still produced; only the recomputation of a known field is skipped.
#include <cuda_fp16.h>

#include "common.cuh"

namespace {

constexpr int TILE = 16;          // must equal conv_tc2.cu T2_H / T2_W

// one block per (frame, tile): out(p) = OR of `in` over the 3x3 window of p (outside the image: 0);
// tile flag = OR of out over the tile's in-image pixels
__global__ void __launch_bounds__(TILE * TILE)
k_bg_layer(const uint8_t *__restrict__ in, int H, int W, int tiles_h, int tiles_w, uint8_t *__restrict__ out,
           int *__restrict__ tile_flag)
{
    const int tile = blockIdx.x;
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, b = tile / (tiles_w * tiles_h);
    const int h = th * TILE + (threadIdx.x >> 4), w = tw * TILE + (threadIdx.x & 15);
    int v = 0;
    if (h < H && w < W) {
        const uint8_t *f = in + (size_t)b * H * W;
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                const int y = h + dy, x = w + dx;
                v |= (y < 0 || y >= H || x < 0 || x >= W) ? 0 : (int)f[(size_t)y * W + x];
            }
        out[((size_t)b * H + h) * W + w] = (uint8_t)(v != 0);
    }
    const int any = __syncthreads_or(v);
    if (threadIdx.x == 0) tile_flag[tile] = any ? 1 : 0;
}

// one block per layer: stable compaction of the tile ids into work (flag 1) and background (flag 0) lists
__global__ void __launch_bounds__(1024)
k_bg_compact(const int *__restrict__ tile_flag, int num_tiles, int *work_list, int *bg_list, int *counts)
{
    const int layer = blockIdx.x;
    const int *flag = tile_flag + (size_t)layer * num_tiles;
    int *work = work_list + (size_t)layer * num_tiles, *bg = bg_list + (size_t)layer * num_tiles;
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < num_tiles; base += 1024) {
        const int i = base + threadIdx.x;
        const int f = i < num_tiles ? flag[i] : 0;
        int total;
        const int ex = b2s_block_exscan(f, &total);
        const int carry = s_carry;
        if (i < num_tiles) {
            if (f) work[carry + ex] = i;
            else bg[i - (carry + ex)] = i;            // background tiles before i: i - (#work tiles before i)
        }
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        counts[2 * layer] = s_carry;
        counts[2 * layer + 1] = num_tiles - s_carry;
    }
}

// one block per background tile (grid-stride): thread = (pixel of a tile row, 16-byte channel chunk), so one load /
// store instruction of the block moves one whole tile row of a plane (16 pixels x 256 B, contiguous in NHWC) from
// the empty-frame response `f` [H+2, W+2, C] to the output map
__global__ void __launch_bounds__(256)
k_bg_fill(const int *__restrict__ bg_list, const int *__restrict__ bg_count, int H, int W, int tiles_h, int tiles_w, int C,
          const __half *__restrict__ f_hi, const __half *__restrict__ f_lo, __half *__restrict__ out_hi,
          __half *__restrict__ out_lo, int out_stride)
{
    const int n = *bg_count;
    const int chunks = C / 8;                         // 16-byte chunks per pixel and plane
    const int px_per_pass = 256 / chunks;             // pixels of a tile row covered per pass (C = 128: 16)
    const int chunk = threadIdx.x % chunks, px = threadIdx.x / chunks;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const int tile = bg_list[i];
        const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, b = tile / (tiles_w * tiles_h);
        for (int r = 0; r < TILE; ++r) {
            const int h = th * TILE + r;
            if (h >= H) break;
            for (int p0 = 0; p0 < TILE; p0 += px_per_pass) {
                const int w = tw * TILE + p0 + px;
                if (p0 + px < TILE && w < W) {
                    const size_t fpix = (size_t)(h + 1) * (W + 2) + (w + 1);
                    const size_t pix = (size_t)b * (H + 2) * (W + 2) + fpix;
                    *reinterpret_cast<uint4 *>(out_hi + pix * out_stride + chunk * 8) =
                        __ldg(reinterpret_cast<const uint4 *>(f_hi + fpix * C + chunk * 8));
                    *reinterpret_cast<uint4 *>(out_lo + pix * out_stride + chunk * 8) =
                        __ldg(reinterpret_cast<const uint4 *>(f_lo + fpix * C + chunk * 8));
                }
            }
        }
    }
}

}  // namespace

extern "C" int b2s_rpn_bg_plan(const uint8_t *occupancy, int batch, int H, int W, int num_layers, uint8_t *scratch,
                               int *tile_flags, int *work_lists, int *bg_lists, int *counts, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(batch >= 1 && H >= 1 && W >= 1 && num_layers >= 1 && num_layers <= 32, "b2s_rpn_bg_plan: bad sizes");
    const int tiles_h = b2s_cdiv(H, TILE), tiles_w = b2s_cdiv(W, TILE);
    const int num_tiles = batch * tiles_h * tiles_w;
    const size_t map = (size_t)batch * H * W;
    const uint8_t *in = occupancy;
    for (int l = 0; l < num_layers; ++l) {
        uint8_t *out = scratch + (size_t)(l & 1) * map;
        k_bg_layer<<<num_tiles, TILE * TILE, 0, stream>>>(in, H, W, tiles_h, tiles_w, out,
                                                          tile_flags + (size_t)l * num_tiles);
        B2S_LAUNCH_OK();
        in = out;
    }
    k_bg_compact<<<num_layers, 1024, 0, stream>>>(tile_flags, num_tiles, work_lists, bg_lists, counts);
    B2S_LAUNCH_OK();
    return 0;
}

extern "C" int b2s_rpn_bg_fill(const int *bg_list, const int *bg_count_dev, int batch, int H, int W, int C,
                               const b2s_half *f_hi, const b2s_half *f_lo, b2s_half *out_hi, b2s_half *out_lo,
                               int out_stride, void *stream_)
{
    cudaStream_t stream = (cudaStream_t)stream_;
    B2S_REQUIRE(C % 8 == 0 && C >= 8 && C <= 2048 && 256 % (C / 8) == 0 && out_stride >= C && out_stride % 8 == 0,
                "b2s_rpn_bg_fill: C must be a multiple of 8 whose chunk count divides 256");
    const int tiles_h = b2s_cdiv(H, TILE), tiles_w = b2s_cdiv(W, TILE);
    const int num_tiles = batch * tiles_h * tiles_w;
    int blocks = num_tiles < 132 * 8 ? num_tiles : 132 * 8;
    k_bg_fill<<<blocks, 256, 0, stream>>>(bg_list, bg_count_dev, H, W, tiles_h, tiles_w, C,
                                          reinterpret_cast<const __half *>(f_hi), reinterpret_cast<const __half *>(f_lo),
                                          reinterpret_cast<__half *>(out_hi), reinterpret_cast<__half *>(out_lo), out_stride);
    B2S_LAUNCH_OK();
    return 0;
}
