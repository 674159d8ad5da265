// pfn_deco.cuh -- the PointPillars feature net's input decoration, shared by the inference kernel (k_pfn, bev.cu) and
// the training kernels (pfn_train.cu), so both see the same fp32 Linear inputs bit for bit.
//
// fp32 op order (every step rounded on its own, no contraction):
//   mean   m = (sum of the pillar's np points' x, y, z, added in slot order from 0.f) / np
//   centre c = (x_index * vx) + x_offset,  (y_index * vy) + y_offset
//   raw    PLAIN: [x, y, z, r, ...];  RADIUS: [sqrt((x * x) + (y * y)), z, r, ...]
//   dec    [x - m.x, y - m.y, z - m.z, x - c.x, y - c.y]
// The Linear input of a point is [raw[0 .. NRAW), dec[0 .. 5)], NRAW = F (PLAIN) or F - 1 (RADIUS).
#pragma once
#include "common.cuh"

struct B2sPfnPillar {
    float mx, my, mz, cx, cy;
};

// mean and centre of one pillar; point(t) -> pointer to slot t's F features
template <class PointAt>
__device__ __forceinline__ B2sPfnPillar b2s_pfn_pillar(PointAt point, int np, int4 q, float vx, float vy, float xoff,
                                                       float yoff)
{
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int t = 0; t < np; ++t) {
        const float *p = point(t);
        sx = __fadd_rn(sx, __ldg(&p[0]));
        sy = __fadd_rn(sy, __ldg(&p[1]));
        sz = __fadd_rn(sz, __ldg(&p[2]));
    }
    const float fn = (float)np;
    B2sPfnPillar g;
    g.mx = __fdiv_rn(sx, fn);
    g.my = __fdiv_rn(sy, fn);
    g.mz = __fdiv_rn(sz, fn);
    g.cx = __fadd_rn(__fmul_rn((float)q.w, vx), xoff);
    g.cy = __fadd_rn(__fmul_rn((float)q.z, vy), yoff);
    return g;
}

// one point's Linear input: raw[0 .. NRAW) and dec[0 .. 5); p holds F <= 8 features
template <int DECO>
__device__ __forceinline__ void b2s_pfn_decorate(const float *p, int F, const B2sPfnPillar &g, float raw[8],
                                                 float dec[5])
{
    float feat[9];
#pragma unroll
    for (int f = 0; f < 9; ++f) feat[f] = (f < F) ? __ldg(&p[f]) : 0.f;
    if (DECO == B2S_PFN_RADIUS) {
        // torch.norm(xy, p=2) with the multiply and add rounded separately, like the mean
        raw[0] = __fsqrt_rn(__fadd_rn(__fmul_rn(feat[0], feat[0]), __fmul_rn(feat[1], feat[1])));
#pragma unroll
        for (int f = 1; f < 8; ++f) raw[f] = feat[f + 1];
    } else {
#pragma unroll
        for (int f = 0; f < 8; ++f) raw[f] = feat[f];
    }
    dec[0] = __fsub_rn(feat[0], g.mx);
    dec[1] = __fsub_rn(feat[1], g.my);
    dec[2] = __fsub_rn(feat[2], g.mz);
    dec[3] = __fsub_rn(feat[0], g.cx);
    dec[4] = __fsub_rn(feat[1], g.cy);
}
