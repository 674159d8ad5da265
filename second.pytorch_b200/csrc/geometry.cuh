// geometry.cuh -- rotated BEV box helpers shared by the NMS / overlap kernels (detect.cu) and the KITTI evaluation
// (kitti_eval.cu).  fp32, as the reference's numba kernels (second/core/non_max_suppression/nms_gpu.py).
#pragma once
#include <math.h>

namespace {

// corners of a BEV box (x,y,w,l,r): clockwise from the min corner, rotated clockwise for positive r
// (second/core/box_np_ops.py:344-357,405-425)
__device__ __forceinline__ void bev_corners(float x, float y, float w, float l, float r, float *c /*8*/)
{
    float s, co;
    sincosf(r, &s, &co);
    const float hx[4] = {-0.5f, -0.5f, 0.5f, 0.5f};
    const float hy[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float px = __fmul_rn(w, hx[i]), py = __fmul_rn(l, hy[i]);
        c[2 * i] = __fadd_rn(__fadd_rn(__fmul_rn(px, co), __fmul_rn(py, s)), x);
        c[2 * i + 1] = __fadd_rn(__fadd_rn(__fmul_rn(-px, s), __fmul_rn(py, co)), y);
    }
}

__device__ __forceinline__ float poly_area(const float *p, int n)
{
    float s = 0.f;
    for (int i = 0; i < n; ++i) {
        int j = (i + 1 == n) ? 0 : i + 1;
        s += p[2 * i] * p[2 * j + 1] - p[2 * j] * p[2 * i + 1];
    }
    return 0.5f * s;
}

// Sutherland-Hodgman clip of convex quad A by convex quad B; returns intersection area (>= 0).
// All eight corners are first taken relative to A's first corner, so the shoelace and clip products stay of the
// size of the pair, not of its position: on raw coordinates near (70, 40) the products are ~2800 against areas of a
// few m^2, and the IoU error grew with the distance from the origin (DESIGN §2).  For a pair far from the origin
// the subtraction is exact (Sterbenz).
__device__ float quad_intersection(const float *a_in, const float *b_in, float *area_a, float *area_b)
{
    float A[8], B[8];
    const float ox = a_in[0], oy = a_in[1];
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
        A[i] = __fsub_rn(a_in[i], ox); A[i + 1] = __fsub_rn(a_in[i + 1], oy);
        B[i] = __fsub_rn(b_in[i], ox); B[i + 1] = __fsub_rn(b_in[i + 1], oy);
    }
    float sa = poly_area(A, 4), sb = poly_area(B, 4);
    if (sa < 0.f) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int j = 3 - i;
            float tx = A[2 * i], ty = A[2 * i + 1];
            A[2 * i] = A[2 * j]; A[2 * i + 1] = A[2 * j + 1];
            A[2 * j] = tx; A[2 * j + 1] = ty;
        }
        sa = -sa;
    }
    if (sb < 0.f) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int j = 3 - i;
            float tx = B[2 * i], ty = B[2 * i + 1];
            B[2 * i] = B[2 * j]; B[2 * i + 1] = B[2 * j + 1];
            B[2 * j] = tx; B[2 * j + 1] = ty;
        }
        sb = -sb;
    }
    *area_a = sa;
    *area_b = sb;
    float buf0[20], buf1[20];
    int n = 4;
#pragma unroll
    for (int i = 0; i < 8; ++i) buf0[i] = A[i];
    float *cur = buf0, *nxt = buf1;
    for (int e = 0; e < 4 && n > 0; ++e) {
        int f = (e + 1) & 3;
        float ax = B[2 * e], ay = B[2 * e + 1], bx = B[2 * f], by = B[2 * f + 1];
        int m = 0;
        for (int i = 0; i < n; ++i) {
            int j = (i + 1 == n) ? 0 : i + 1;
            float px = cur[2 * i], py = cur[2 * i + 1], qx = cur[2 * j], qy = cur[2 * j + 1];
            float sp = (bx - ax) * (py - ay) - (by - ay) * (px - ax);
            float sq = (bx - ax) * (qy - ay) - (by - ay) * (qx - ax);
            bool pin = sp >= 0.f, qin = sq >= 0.f;
            if (pin) { nxt[2 * m] = px; nxt[2 * m + 1] = py; ++m; }
            if (pin != qin) {
                float t = sp / (sp - sq);
                nxt[2 * m] = px + t * (qx - px);
                nxt[2 * m + 1] = py + t * (qy - py);
                ++m;
            }
        }
        n = m;
        float *tmp = cur; cur = nxt; nxt = tmp;
    }
    if (n < 3) return 0.f;
    float inter = poly_area(cur, n);
    return inter > 0.f ? inter : 0.f;
}

__device__ __forceinline__ void standup_of(const float *c, float *s /*x1,y1,x2,y2*/)
{
    s[0] = fminf(fminf(c[0], c[2]), fminf(c[4], c[6]));
    s[1] = fminf(fminf(c[1], c[3]), fminf(c[5], c[7]));
    s[2] = fmaxf(fmaxf(c[0], c[2]), fmaxf(c[4], c[6]));
    s[3] = fmaxf(fmaxf(c[1], c[3]), fmaxf(c[5], c[7]));
}

}  // namespace
