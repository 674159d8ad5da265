// box_geom.cuh -- box geometry shared by the training kernels (augment.cu, dbsample.cu), in the reference's dtypes
// and step order (box_np_ops.py / preprocess.py / geometry.py of second):
//   Ar<T>          round-to-nearest arithmetic in float32 or float64, so --fmad=true cannot contract a step;
//   box_planes     center_to_corner_box3d(origin = 0.5) -> corner_to_surfaces_3d -> surface_equ_3d_jitv2, the planes
//                  points_in_convex_polygon_3d_jit tests (a point is inside when every plane gives a negative value);
//   corners2d      box2d_to_corner_jit / center_to_corner_box2d of (x, y, w, l, r), with standup its bounding box;
//   collide        box_collision_test of one (boxes row, qboxes column) pair.
#pragma once
#include <math.h>

#include "common.cuh"

namespace {

template <typename T> struct Ar;
template <> struct Ar<float> {
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
    static __device__ __forceinline__ float from(double a) { return __double2float_rn(a); }
    // the float64 function rounded once: within an ulp of numba's / numpy's float32 sin and cos, and reproducible
    static __device__ __forceinline__ float sin_(float a) { return __double2float_rn(sin((double)a)); }
    static __device__ __forceinline__ float cos_(float a) { return __double2float_rn(cos((double)a)); }
};
template <> struct Ar<double> {
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
    static __device__ __forceinline__ double from(double a) { return a; }
    static __device__ __forceinline__ double sin_(double a) { return sin(a); }
    static __device__ __forceinline__ double cos_(double a) { return cos(a); }
};

// a += b with a of dtype T and b float64: numpy adds in float64 and rounds once
template <typename T>
__device__ __forceinline__ T add_f64(T a, double b) { return Ar<T>::from(__dadd_rn((double)a, b)); }

// float32 point coordinate op T box value, in the promoted dtype, stored through float32
__device__ __forceinline__ float pt_sub(float p, float c) { return __fsub_rn(p, c); }
__device__ __forceinline__ float pt_sub(float p, double c) { return __double2float_rn(__dsub_rn((double)p, c)); }
__device__ __forceinline__ float pt_add(float p, float c) { return __fadd_rn(p, c); }
__device__ __forceinline__ float pt_add(float p, double c) { return __double2float_rn(__dadd_rn((double)p, c)); }

// (x, y) @ [[c, -s], [s, c]] -- the reference's row-vector rotation, each product rounded, then summed
template <typename T>
__device__ __forceinline__ void rot2(T &x, T &y, T c, T s)
{
    using M = Ar<T>;
    const T nx = M::add(M::mul(x, c), M::mul(y, s));
    const T ny = M::add(M::mul(x, -s), M::mul(y, c));
    x = nx;
    y = ny;
}

// center_to_corner_box3d(origin = 0.5, axis = 2) -> corner_to_surfaces_3d_jit -> surface_equ_3d_jitv2
template <typename T>
__device__ void box_planes(const T *b, T *out)
{
    using M = Ar<T>;
    // corners_nd's order: x0y0z0, x0y0z1, x0y1z1, x0y1z0, x1y0z0, x1y0z1, x1y1z1, x1y1z0
    const int cx[8] = {0, 0, 0, 0, 1, 1, 1, 1}, cy[8] = {0, 0, 1, 1, 0, 0, 1, 1}, cz[8] = {0, 1, 1, 0, 0, 1, 1, 0};
    const T c = M::cos_(b[6]), s = M::sin_(b[6]);
    T cr[8][3];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        T x = M::mul(b[3], cx[k] ? T(0.5) : T(-0.5));
        T y = M::mul(b[4], cy[k] ? T(0.5) : T(-0.5));
        const T z = M::mul(b[5], cz[k] ? T(0.5) : T(-0.5));
        rot2<T>(x, y, c, s);                       // einsum with rot_mat_T [[c, -s, 0], [s, c, 0], [0, 0, 1]]
        cr[k][0] = M::add(x, b[0]);
        cr[k][1] = M::add(y, b[1]);
        cr[k][2] = M::add(z, b[2]);
    }
    const int idx[6][3] = {{0, 1, 2}, {7, 6, 5}, {0, 3, 7}, {1, 5, 6}, {0, 4, 5}, {3, 2, 6}};
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        const T *s0 = cr[idx[j][0]], *s1 = cr[idx[j][1]], *s2 = cr[idx[j][2]];
        const T a0 = M::sub(s0[0], s1[0]), a1 = M::sub(s0[1], s1[1]), a2 = M::sub(s0[2], s1[2]);
        const T b0 = M::sub(s1[0], s2[0]), b1 = M::sub(s1[1], s2[1]), b2 = M::sub(s1[2], s2[2]);
        const T n0 = M::sub(M::mul(a1, b2), M::mul(a2, b1));
        const T n1 = M::sub(M::mul(a2, b0), M::mul(a0, b2));
        const T n2 = M::sub(M::mul(a0, b1), M::mul(a1, b0));
        const T d = M::sub(M::sub(M::mul(-s0[0], n0), M::mul(s0[1], n1)), M::mul(s0[2], n2));
        out[j * 4 + 0] = n0;
        out[j * 4 + 1] = n1;
        out[j * 4 + 2] = n2;
        out[j * 4 + 3] = d;
    }
}

// box2d_to_corner_jit of (x, y, w, l, r)
template <typename T>
__device__ __forceinline__ void corners2d(T x, T y, T w, T l, T r, T out[8])
{
    using M = Ar<T>;
    const T c = M::cos_(r), s = M::sin_(r);
    const T nx[4] = {T(-0.5), T(-0.5), T(0.5), T(0.5)}, ny[4] = {T(-0.5), T(0.5), T(0.5), T(-0.5)};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        T px = M::mul(w, nx[k]), py = M::mul(l, ny[k]);
        rot2<T>(px, py, c, s);
        out[2 * k] = M::add(px, x);
        out[2 * k + 1] = M::add(py, y);
    }
}

template <typename T>
__device__ __forceinline__ void standup(const T c[8], T su[4])
{
    su[0] = fmin(fmin(c[0], c[2]), fmin(c[4], c[6]));
    su[1] = fmin(fmin(c[1], c[3]), fmin(c[5], c[7]));
    su[2] = fmax(fmax(c[0], c[2]), fmax(c[4], c[6]));
    su[3] = fmax(fmax(c[1], c[3]), fmax(c[5], c[7]));
}

// every corner of q strictly inside the clockwise quad a (cross < 0 for all edges)
template <typename T>
__device__ __forceinline__ bool contains(const T *a, const T *q)
{
    using M = Ar<T>;
    for (int l = 0; l < 4; ++l) {
        for (int k = 0; k < 4; ++k) {
            const int k1 = (k + 1) & 3;
            const T v0 = -M::sub(a[2 * k], a[2 * k1]), v1 = -M::sub(a[2 * k + 1], a[2 * k1 + 1]);
            T cross = M::mul(v1, M::sub(a[2 * k], q[2 * l]));
            cross = M::sub(cross, M::mul(v0, M::sub(a[2 * k + 1], q[2 * l + 1])));
            if (cross >= T(0)) return false;
        }
    }
    return true;
}

// box_collision_test of one pair, its predicates in the box dtype
template <typename T>
__device__ bool collide(const T *a, const T *asu, const T *q, const T *qsu)
{
    using M = Ar<T>;
    const T iw = M::sub(fmin(asu[2], qsu[2]), fmax(asu[0], qsu[0]));
    if (!(iw > T(0))) return false;
    const T ih = M::sub(fmin(asu[3], qsu[3]), fmax(asu[1], qsu[1]));
    if (!(ih > T(0))) return false;
    for (int k = 0; k < 4; ++k) {
        const T A0 = a[2 * k], A1 = a[2 * k + 1], B0 = a[2 * ((k + 1) & 3)], B1 = a[2 * ((k + 1) & 3) + 1];
        for (int l = 0; l < 4; ++l) {
            const T C0 = q[2 * l], C1 = q[2 * l + 1], D0 = q[2 * ((l + 1) & 3)], D1 = q[2 * ((l + 1) & 3) + 1];
            const bool acd = M::mul(M::sub(D1, A1), M::sub(C0, A0)) > M::mul(M::sub(C1, A1), M::sub(D0, A0));
            const bool bcd = M::mul(M::sub(D1, B1), M::sub(C0, B0)) > M::mul(M::sub(C1, B1), M::sub(D0, B0));
            if (acd != bcd) {
                const bool abc = M::mul(M::sub(C1, A1), M::sub(B0, A0)) > M::mul(M::sub(B1, A1), M::sub(C0, A0));
                const bool abd = M::mul(M::sub(D1, A1), M::sub(B0, A0)) > M::mul(M::sub(B1, A1), M::sub(D0, A0));
                if (abc != abd) return true;
            }
        }
    }
    return contains<T>(a, q) || contains<T>(q, a);
}

// points_in_convex_polygon_3d_jit of one float32 point against one box's planes (box_planes' layout)
template <typename T>
__device__ __forceinline__ bool in_planes(const T *pl, float x, float y, float z)
{
    using M = Ar<T>;
    for (int j = 0; j < 6; ++j) {
        const T sign = M::add(M::add(M::add(M::mul(T(x), pl[4 * j]), M::mul(T(y), pl[4 * j + 1])),
                                     M::mul(T(z), pl[4 * j + 2])), pl[4 * j + 3]);
        if (!(sign < T(0))) return false;
    }
    return true;
}

}  // namespace
