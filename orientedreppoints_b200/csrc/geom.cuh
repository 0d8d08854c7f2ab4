// geom.cuh - device-side rotated-quadrilateral geometry for sm_90a.
//
// Two IoU evaluators live here:
//
//  (1) ref_quad_pair<T>   the reference's algorithm - signed triangle fan about the origin, three
//      half-plane cuts per triangle pair - in T = double (DOTA_devkit/polyiou.cpp:58-128) or
//      T = float (mmdet/ops/nms/src/rnms_kernel.cu:17-147 == DOTA_devkit/poly_nms_gpu/
//      poly_nms_kernel.cu:31-212).  Every operation goes through the round-to-nearest intrinsics
//      (__fmul_rn, __dadd_rn, ...) which nvcc never contracts into FMAs, so the results are
//      bit-identical to the reference's x86-64 builds (no FMA there either).
//
//  (2) fast_quad_pair     Sutherland-Hodgman clipping of quad A by the four half-planes of quad B in
//      PAIR-LOCAL coordinates (fp32).  It returns the intersection, both areas and a bound on the
//      absolute error of those numbers; callers that need a decision (`iou > thr`) fall back to (1)
//      in double whenever the decision margin is inside the bound, so decisions always equal the
//      fp64 reference's.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace orp {

// ---------------------------------------------------------------------------------------------
// exactly-rounded arithmetic (never contracted)
// ---------------------------------------------------------------------------------------------
template <typename T> struct Rn;
template <> struct Rn<float> {
    static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
    static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
    static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
    static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
    static __device__ __forceinline__ int sgn(float v) { return (v > 1E-8f) - (v < -1E-8f); }
};
template <> struct Rn<double> {
    static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
    static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
    static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
    static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
    static __device__ __forceinline__ int sgn(double v) { return (v > 1E-8) - (v < -1E-8); }
};

template <typename T> struct Pt { T x, y; };

template <typename T>
__device__ __forceinline__ bool pt_same(Pt<T> a, Pt<T> b)
{
    return Rn<T>::sgn(Rn<T>::sub(a.x, b.x)) == 0 && Rn<T>::sgn(Rn<T>::sub(a.y, b.y)) == 0;
}

template <typename T>
__device__ __forceinline__ T cross3(Pt<T> o, Pt<T> a, Pt<T> b)
{
    using R = Rn<T>;
    T l = R::mul(R::sub(a.x, o.x), R::sub(b.y, o.y));
    T r = R::mul(R::sub(b.x, o.x), R::sub(a.y, o.y));
    return R::sub(l, r);
}

// shoelace of ring v[0..n-1]; v must have room for the sentinel v[n]
template <typename T>
__device__ __forceinline__ T ring_area(Pt<T> *v, int n)
{
    using R = Rn<T>;
    T acc = 0;
    v[n] = v[0];
    for (int i = 0; i < n; ++i) {
        T t = R::sub(R::mul(v[i].x, v[i + 1].y), R::mul(v[i].y, v[i + 1].x));
        acc = R::add(acc, t);
    }
    return acc * (T)0.5;  // exact
}

constexpr int kRingCap = 9;   // a triangle cut three times has <= 6 vertices (+ sentinel)
constexpr int kTmpCap = 14;

// keep the part of ring v strictly left of a->b (reference polygon_cut)
template <typename T>
__device__ __forceinline__ int half_plane_cut(Pt<T> *v, int n, Pt<T> a, Pt<T> b, Pt<T> *tmp)
{
    using R = Rn<T>;
    int m = 0;
    v[n] = v[0];
    T cprev = cross3(a, b, v[0]);
    for (int i = 0; i < n; ++i) {
        T cnext = cross3(a, b, v[i + 1]);
        int si = R::sgn(cprev), sj = R::sgn(cnext);
        if (si > 0 && m < kTmpCap) tmp[m++] = v[i];
        if (si != sj) {
            // reference lineCross: s1 = cross(a,b,c), s2 = cross(a,b,d)
            T s1 = cprev, s2 = cnext;
            if (!(R::sgn(s1) == 0 && R::sgn(s2) == 0)) {
                T den = R::sub(s2, s1);
                if (R::sgn(den) != 0 && m < kTmpCap) {
                    tmp[m].x = R::div(R::sub(R::mul(v[i].x, s2), R::mul(v[i + 1].x, s1)), den);
                    tmp[m].y = R::div(R::sub(R::mul(v[i].y, s2), R::mul(v[i + 1].y, s1)), den);
                }
            }
            if (m < kTmpCap) ++m;
        }
        cprev = cnext;
    }
    int k = 0;
    for (int i = 0; i < m; ++i)
        if (i == 0 || !pt_same(tmp[i], tmp[i - 1])) { if (k < kRingCap - 1) v[k++] = tmp[i]; }
    while (k > 1 && pt_same(v[k - 1], v[0])) --k;
    return k;
}

// ABS = false: convex_iou_kernel.cu:124-127 keeps the sign of the clipped triangle's area (polyiou.cpp:86 takes fabs)
template <typename T, bool ABS = true>
__device__ __forceinline__ T fan_pair(Pt<T> a, Pt<T> b, Pt<T> c, Pt<T> d)
{
    using R = Rn<T>;
    Pt<T> o{(T)0, (T)0};
    int s1 = R::sgn(cross3(o, a, b));
    int s2 = R::sgn(cross3(o, c, d));
    if (s1 == 0 || s2 == 0) return (T)0;
    if (s1 < 0) { Pt<T> t = a; a = b; b = t; }
    if (s2 < 0) { Pt<T> t = c; c = d; d = t; }
    Pt<T> ring[kRingCap];
    Pt<T> tmp[kTmpCap];
#pragma unroll
    for (int i = 0; i < kTmpCap; ++i) { tmp[i].x = 0; tmp[i].y = 0; }
    ring[0] = o; ring[1] = a; ring[2] = b;
    int n = 3;
    n = half_plane_cut(ring, n, o, c, tmp);
    n = half_plane_cut(ring, n, c, d, tmp);
    n = half_plane_cut(ring, n, d, o, tmp);
    T ar = ring_area(ring, n);
    if (ABS) ar = ar < 0 ? -ar : ar;
    return (s1 * s2 == -1) ? -ar : ar;
}

template <typename T> struct PairRes { T inter, area_p, area_q; };

// p, q: 8 coordinates each (x1,y1,...,x4,y4) already converted to T
template <typename T>
__device__ __noinline__ PairRes<T> ref_quad_pair(const T *p, const T *q)
{
    using R = Rn<T>;
    Pt<T> A[6], B[6];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        A[i].x = p[2 * i]; A[i].y = p[2 * i + 1];
        B[i].x = q[2 * i]; B[i].y = q[2 * i + 1];
    }
    if (ring_area(A, 4) < 0) { Pt<T> t = A[0]; A[0] = A[3]; A[3] = t; t = A[1]; A[1] = A[2]; A[2] = t; }
    if (ring_area(B, 4) < 0) { Pt<T> t = B[0]; B[0] = B[3]; B[3] = t; t = B[1]; B[1] = B[2]; B[2] = t; }
    A[4] = A[0]; B[4] = B[0];
    T acc = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) acc = R::add(acc, fan_pair(A[i], A[i + 1], B[j], B[j + 1]));
    PairRes<T> r;
    r.inter = acc;
    T ap = ring_area(A, 4), aq = ring_area(B, 4);
    r.area_p = ap < 0 ? -ap : ap;
    r.area_q = aq < 0 ? -aq : aq;
    return r;
}

// iou from a PairRes under the three zero-union conventions (see orp_b200.h)
template <typename T>
__device__ __forceinline__ T iou_from(const PairRes<T> &r, int union_mode)
{
    using R = Rn<T>;
    T uni = R::sub(R::add(r.area_p, r.area_q), r.inter);
    if (union_mode == ORP_UNION_GUARD && uni == 0) return R::div(R::add(r.inter, (T)1), R::add(uni, (T)1));
    return R::div(r.inter, uni);
}

// does an IoU value suppress under `iou > thr` / `!(iou <= thr)` ?
template <typename T>
__device__ __forceinline__ bool suppresses(T iou, T thr, int union_mode)
{
    if (union_mode == ORP_UNION_NAN_SUPPRESSES || union_mode == ORP_UNION_NAN_SUPPRESSES_ALL) return !(iou <= thr);
    return iou > thr;
}

// ---------------------------------------------------------------------------------------------
// fast path: Sutherland-Hodgman in pair-local fp32 coordinates
// ---------------------------------------------------------------------------------------------
// The fast path clips a CONVEX subject by a CONVEX window.  The reference algorithm accepts any
// quadrilateral (concave, self-intersecting: it integrates a signed measure), so anything that is
// not a convex quadrilateral with positive area is routed to ref_quad_pair<double> instead.
__device__ __forceinline__ bool quad_is_convex(const float *c)
{
    bool pos = true, neg = true, any = false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int a = k, b = (k + 1) & 3, d = (k + 2) & 3;
        const float ux = c[2 * b] - c[2 * a], uy = c[2 * b + 1] - c[2 * a + 1];
        const float vx = c[2 * d] - c[2 * b], vy = c[2 * d + 1] - c[2 * b + 1];
        const float z = ux * vy - uy * vx;
        pos = pos && (z >= 0.f);
        neg = neg && (z <= 0.f);
        any = any || (z != 0.f);
    }
    return (pos || neg) && any;
}

struct FastRes {
    float inter, area_a, area_b;  // absolute areas
    float err;                    // bound on the absolute error of each of the three numbers
};

// a[8], b[8]: quads already translated to a pair-local origin.  FMAs allowed here.
template <int S>
__device__ __forceinline__ FastRes fast_quad_pair_s(const float *a, const float *b, float *w)
{
    float ax[4], ay[4], bx[4], by[4];
    float L = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        ax[i] = a[2 * i]; ay[i] = a[2 * i + 1];
        bx[i] = b[2 * i]; by[i] = b[2 * i + 1];
        L = fmaxf(L, fmaxf(fmaxf(fabsf(ax[i]), fabsf(ay[i])), fmaxf(fabsf(bx[i]), fabsf(by[i]))));
    }
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int j = (i + 1) & 3;
        sa += ax[i] * ay[j] - ay[i] * ax[j];
        sb += bx[i] * by[j] - by[i] * bx[j];
    }
    // orient B counter-clockwise (inside = left of each edge); A's orientation is irrelevant
    if (sb < 0.f) {
        float t;
        t = bx[0]; bx[0] = bx[3]; bx[3] = t; t = by[0]; by[0] = by[3]; by[3] = t;
        t = bx[1]; bx[1] = bx[2]; bx[2] = t; t = by[1]; by[1] = by[2]; by[2] = t;
    }
    // two ping-pong vertex rings of <= 9 points in the caller's scratch (element k of array j at w[(j*10 + k) * S]):
    // shared memory with S = blockDim for the NMS sweep (no local-memory traffic), a local array with S = 1 elsewhere
    int n = 4, src = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) { w[(0 * 10 + i) * S] = ax[i]; w[(1 * 10 + i) * S] = ay[i]; }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (n == 0) break;
        const float ex = bx[(k + 1) & 3] - bx[k], ey = by[(k + 1) & 3] - by[k];
        const float ox = bx[k], oy = by[k];
        float *sx = w + (src * 20) * S, *sy = w + (src * 20 + 10) * S;
        float *dx = w + ((src ^ 1) * 20) * S, *dy = w + ((src ^ 1) * 20 + 10) * S;
        int m = 0;
        const float fx = sx[0], fy = sy[0];
        float cx = fx, cy = fy;
        float dc = ex * (cy - oy) - ey * (cx - ox);
        for (int i = 0; i < n; ++i) {
            const bool last = (i + 1 == n);
            const float nx = last ? fx : sx[(i + 1) * S], ny = last ? fy : sy[(i + 1) * S];
            const float dn = ex * (ny - oy) - ey * (nx - ox);
            const bool inc = dc >= 0.f, inn = dn >= 0.f;
            if (inc) { dx[m * S] = cx; dy[m * S] = cy; ++m; }
            if (inc != inn) {
                const float t = dc / (dc - dn);
                dx[m * S] = fmaf(t, nx - cx, cx);
                dy[m * S] = fmaf(t, ny - cy, cy);
                ++m;
            }
            cx = nx; cy = ny; dc = dn;
        }
        n = m < 9 ? m : 9;
        src ^= 1;
    }
    float si = 0.f;
    if (n > 0) {
        const float *sx = w + (src * 20) * S, *sy = w + (src * 20 + 10) * S;
        const float fx = sx[0], fy = sy[0];
        float cx = fx, cy = fy;
        for (int i = 0; i < n; ++i) {
            const bool last = (i + 1 == n);
            const float nx = last ? fx : sx[(i + 1) * S], ny = last ? fy : sy[(i + 1) * S];
            si += cx * ny - cy * nx;
            cx = nx; cy = ny;
        }
    }
    FastRes r;
    r.inter = 0.5f * fabsf(si);
    r.area_a = 0.5f * fabsf(sa);
    r.area_b = 0.5f * fabsf(sb);
    // |coords| <= L: every cross product carries <= ~4 eps L^2, intersection points <= ~8 eps L,
    // a <=8-gon shoelace sums 8 of them.  64 eps L^2 is a generous envelope (validated empirically
    // in tests/test_nms_gpu.py::test_fast_clip_error_envelope).
    r.err = 64.f * 5.9604645e-08f * L * L;
    return r;
}

// convenience form with thread-local scratch
__device__ __forceinline__ FastRes fast_quad_pair(const float *a, const float *b)
{
    float w[40];
    return fast_quad_pair_s<1>(a, b, w);
}

}  // namespace orp
