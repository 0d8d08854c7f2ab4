// convex_iou.cu - IoU between the convex hull of a 9-point set and a quadrilateral (SURVEY §8 row n2).
// Replaces mmdet/ops/iou/src/convex_iou_kernel.cu:268-312 (convex_iou_kernel / devrIoU) and its host wrapper
// :315-360 (blocking cudaMemcpy to the host, element loop, .to(device)): the result stays on the device.
//
// Arithmetic: fp64, every operation separately rounded (the CPU oracle's sequence), float result.
// One thread per (point set, quadrilateral) pair; the hull (a few dozen cross products) is rebuilt per pair, which
// keeps all pairs independent - the clipping of 4 x (hull edges) triangle pairs dominates.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "geom.cuh"

namespace orp {
namespace {

using P = Pt<double>;

__device__ __forceinline__ double dist2(P a, P b)
{
    const double dx = __dsub_rn(a.x, b.x), dy = __dsub_rn(a.y, b.y);
    return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
}

// Jarvis_and_index (convex_iou_kernel.cu:139-266; convex_giou_kernel.cu:618-728) and Jarvis (convex_giou_kernel.cu:454-542):
// gift wrapping of v[0..n-1] (n <= NMAX, v with room for 2 * NMAX + 2 points) in place from the lowest point, right chain
// (turn > 0, ties -> the farther point) then left chain (turn < 0).  Chains are bounded at n + 1 steps, where the reference
// loops forever (NaN input); `closed` tells whether both chains reached the top point.
template <int NMAX>
__device__ int jarvis(P *v, int n, bool &closed)
{
    P pmax = v[0];
    int imax = 0;
    for (int i = 0; i < n; ++i) {
        if (v[i].y < v[0].y || (v[i].y == v[0].y && v[i].x < v[0].x)) { P t = v[0]; v[0] = v[i]; v[i] = t; }
        if (i == 0) { pmax = v[0]; imax = 0; }
        if (v[i].y > pmax.y || (v[i].y == pmax.y && v[i].x > pmax.x)) { pmax = v[i]; imax = i; }
    }
    if (imax == 0) { imax = 1; pmax = v[1]; }
    int st[2][NMAX + 3], top[2];
    closed = true;
    for (int dir = 0; dir < 2; ++dir) {
        int t = 0, k = 0;
        st[dir][0] = 0;
        while (k != imax && t < n + 1) {
            P pk = pmax;
            k = imax;
            const P base = v[st[dir][t]];
            for (int i = 1; i < n; ++i) {
                const double s = cross3(base, v[i], pk);
                const bool take = dir ? (s < 0) : (s > 0);
                if (take || (s == 0 && dist2(base, v[i]) > dist2(base, pk))) { pk = v[i]; k = i; }
            }
            st[dir][++t] = k;
        }
        closed = closed && k == imax;
        top[dir] = t;
    }
    P out[2 * NMAX + 2];
    const int nh = top[0] + top[1];
    for (int i = 0; i < nh; ++i) out[i] = (i <= top[0]) ? v[st[0][i]] : v[st[1][top[1] - (i - top[0])]];
    for (int i = 0; i < nh; ++i) v[i] = out[i];
    return nh;
}

__device__ int hull9(P *v /* in: 9 points, out: ring */)
{
    bool closed;
    return jarvis<9>(v, 9, closed);
}

__device__ __forceinline__ void reverse_ring(P *v, int n)
{
    for (int i = 0, j = n - 1; i < j; ++i, --j) { P t = v[i]; v[i] = v[j]; v[j] = t; }
}

__global__ void __launch_bounds__(128)
convex_iou_kernel(const float *__restrict__ pts, int n, const float *__restrict__ quads, int k, float *__restrict__ out)
{
    const size_t total = (size_t)n * k;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(idx / k), j = (int)(idx - (size_t)i * k);
        P A[26], B[6];
        for (int t = 0; t < 9; ++t) { A[t].x = (double)pts[(size_t)i * 18 + 2 * t]; A[t].y = (double)pts[(size_t)i * 18 + 2 * t + 1]; }
        int n1 = hull9(A);
        for (int t = 0; t < 4; ++t) { B[t].x = (double)quads[(size_t)j * 8 + 2 * t]; B[t].y = (double)quads[(size_t)j * 8 + 2 * t + 1]; }
        // devrIoU, convex_iou_kernel.cu:268-294 with intersectAreaO :126-137
        if (ring_area(A, n1) < 0) reverse_ring(A, n1);
        if (ring_area(B, 4) < 0) reverse_ring(B, 4);
        A[n1] = A[0]; B[4] = B[0];
        double inter = 0;
        for (int a = 0; a < n1; ++a)
            for (int b = 0; b < 4; ++b) inter = __dadd_rn(inter, fan_pair<double, false>(A[a], A[a + 1], B[b], B[b + 1]));
        const double sp = ring_area(A, n1), sq = ring_area(B, 4);
        const double uni = __dsub_rn(__dadd_rn(fabs(sp), fabs(sq)), inter);
        out[idx] = (float)__ddiv_rn(inter, uni);
    }
}

// ---------------------------------------------------------------------------------------------------------- convex_giou
// devrIoU of convex_giou_kernel.cu:730-804 and everything it calls, in the reference's operation order.
//
// Bounds.  A triangle (o, a, b) cut by the three half-planes of intersectArea keeps at most 4 vertices in exact arithmetic;
// the reference stores each cut's Jacobian in [10][10] matrices (<= 5 vertices) and each cut's pre-deduplication rows in
// ccur_grad[100] (k inputs x m rows: 4 k m <= 100).  Inputs beyond those arrays are outside what the reference defines;
// the device flags them and writes a NaN row (DESIGN deviation 13).  The union hull takes at most 9 + 4 points.
constexpr int kCutOut = 5;    // vertices after one cut
constexpr int kCutRows = 8;   // rows before deduplication: k >= 3 inputs and 4 k m <= 100
constexpr int kUnionMax = 13;

// d(cut vertex v) / d(input vertex src[v][e]) as the 2x2 block blk[v][e][c], c in the reference's cut_grad order
// (dx/dx, dy/dx, dx/dy, dy/dy); a vertex depends on at most two inputs, every other entry is +0 as in the reference
struct CutJac {
    int src[kCutRows][2];
    double blk[kCutRows][2][4];
};

__device__ __forceinline__ double jac_at(const CutJac &J, int r, int c)
{
    const int v = r >> 1, s = c >> 1, e = ((c & 1) << 1) | (r & 1);
    if (J.src[v][0] == s) return J.blk[v][0][e];
    if (J.src[v][1] == s) return J.blk[v][1][e];
    return 0.0;
}

// polygon_cut + lineCross (convex_giou_kernel.cu:122-211): keep the part of ring p[0..n-1] strictly left of a->b and the
// Jacobian of the new ring.  Where the reference reads an uninitialised point (one endpoint within 1e-8 of the line, the
// other within 1e-8 of it: lineCross returns without writing) the device takes the endpoint on the line, with a zero row.
__device__ int cut_grad(P *p, int n, P a, P b, CutJac &J, bool &bad)
{
    P pp[kCutRows];
    const int k = n;
    int m = 0;
    p[n] = p[0];
    double cc = cross3(a, b, p[0]);
    for (int i = 0; i < n && !bad; ++i) {
        const double cn = cross3(a, b, p[i + 1]);
        const int si = Rn<double>::sgn(cc), sj = Rn<double>::sgn(cn);
        if (si > 0) {
            if (4 * k * (m + 1) > 100) { bad = true; break; }
            pp[m] = p[i];
            J.src[m][0] = i; J.src[m][1] = -1;
            J.blk[m][0][0] = 1.0; J.blk[m][0][1] = 0.0; J.blk[m][0][2] = 0.0; J.blk[m][0][3] = 1.0;
            ++m;
        }
        if (si != sj) {
            if (4 * k * (m + 1) > 100) { bad = true; break; }
            const P c = p[i], d = p[i + 1];
            const double s1 = cc, s2 = cn;
            const double D = __dsub_rn(s2, s1);
            J.src[m][0] = -1; J.src[m][1] = -1;
            if (Rn<double>::sgn(D) == 0) {
                pp[m] = si == 0 ? c : d;
            } else {
                const double d1x = -__dsub_rn(b.y, a.y), d1y = __dsub_rn(b.x, a.x);   // ds1/dxc, ds1/dyc = ds2/dxd, ds2/dyd
                const double D2 = __dmul_rn(D, D);
                const double X = __dsub_rn(__dmul_rn(c.x, s2), __dmul_rn(d.x, s1));
                const double Y = __dsub_rn(__dmul_rn(c.y, s2), __dmul_rn(d.y, s1));
                double *gc = J.blk[m][0], *gd = J.blk[m][1];
                gc[0] = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(s2, __dmul_rn(d.x, d1x)), D), __dmul_rn(X, -d1x)), D2);
                gc[2] = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(0.0, __dmul_rn(d.x, d1y)), D), __dmul_rn(X, -d1y)), D2);
                gd[0] = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(__dmul_rn(c.x, d1x), s1), D), __dmul_rn(X, d1x)), D2);
                gd[2] = __ddiv_rn(__dsub_rn(__dmul_rn(__dmul_rn(c.x, d1y), D), __dmul_rn(X, d1y)), D2);
                gc[1] = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(0.0, __dmul_rn(d.y, d1x)), D), __dmul_rn(Y, -d1x)), D2);
                gc[3] = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(s2, __dmul_rn(d.y, d1y)), D), __dmul_rn(Y, -d1y)), D2);
                gd[1] = __ddiv_rn(__dsub_rn(__dmul_rn(__dmul_rn(c.y, d1x), D), __dmul_rn(Y, d1x)), D2);
                gd[3] = __ddiv_rn(__dsub_rn(__dmul_rn(__dsub_rn(__dmul_rn(c.y, d1y), s1), D), __dmul_rn(Y, d1y)), D2);
                pp[m].x = __ddiv_rn(X, D);
                pp[m].y = __ddiv_rn(Y, D);
                J.src[m][0] = i;
                J.src[m][1] = i == n - 1 ? 0 : i + 1;
            }
            ++m;
        }
        cc = cn;
    }
    if (bad) return 0;
    int r = 0;
    for (int i = 0; i < m; ++i) {
        if (i == 0 || !pt_same(pp[i], pp[i - 1])) {
            p[r] = pp[i];
            J.src[r][0] = J.src[i][0]; J.src[r][1] = J.src[i][1];
            for (int e = 0; e < 2; ++e)
                for (int c = 0; c < 4; ++c) J.blk[r][e][c] = J.blk[i][e][c];
            ++r;
        }
    }
    while (r > 1 && pt_same(p[r - 1], p[0])) --r;
    if (r > kCutOut) bad = true;
    return r;
}

// polygen_area_grad with the identity map (convex_giou_kernel.cu:73-120): shoelace area of ring p[0..n-1] and its gradient
// g[2v], g[2v+1] with respect to vertex v
__device__ double area_grad(P *p, int n, double *g)
{
    p[n] = p[0];
    double res = 0;
    for (int i = 0; i < n; ++i) res = __dadd_rn(res, __dsub_rn(__dmul_rn(p[i].x, p[i + 1].y), __dmul_rn(p[i].y, p[i + 1].x)));
    for (int v = 0; v < n; ++v) {
        const P prev = p[v == 0 ? n - 1 : v - 1], next = p[v + 1];
        g[2 * v] = __ddiv_rn(__dadd_rn(-prev.y, next.y), 2.0);
        g[2 * v + 1] = __ddiv_rn(__dadd_rn(prev.x, -next.x), 2.0);
    }
    return __ddiv_rn(res, 2.0);
}

// intersectArea (convex_giou_kernel.cu:213-438): signed area of triangle (o, a, b) inside triangle (o, c, d); adds its
// gradient with respect to a and b to ring vertices `order` and `order + 1` (mod cn) of gAB.  The chain-rule products sum
// over the reference's full index ranges, zero entries included (0 * inf is NaN).
__device__ double tri_pair_grad(P a, P b, P c, P d, double *gAB, int order, int cn, bool &bad)
{
    const P o{0.0, 0.0};
    const int s1 = Rn<double>::sgn(cross3(o, a, b)), s2 = Rn<double>::sgn(cross3(o, c, d));
    if (s1 == 0 || s2 == 0) return 0.0;
    const bool flip = s1 == -1;
    if (flip) { P t = a; a = b; b = t; }
    if (s2 == -1) { P t = c; c = d; d = t; }
    P ring[kCutRows + 1];
    ring[0] = o; ring[1] = a; ring[2] = b;
    CutJac J1, J2, J3;
    const int n1 = cut_grad(ring, 3, o, c, J1, bad);
    const int n2 = cut_grad(ring, n1, c, d, J2, bad);
    const int n3 = cut_grad(ring, n2, d, o, J3, bad);
    if (bad) return 0.0;
    double gp[2 * kCutOut];
    double res = area_grad(ring, n3, gp);
    const bool neg = s1 * s2 == -1;
    // p3_p1 = p3_p2 * p2_p1 and p3_p = p3_p1 * p1_p, one row at a time; S_grad sums the rows in order
    double S[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = 0; i < 2 * n3; ++i) {
        double r31[2 * kCutOut];
        for (int j = 0; j < 2 * n1; ++j) {
            double sum = 0.0;
            for (int m = 0; m < 2 * n2; ++m) sum = __dadd_rn(sum, __dmul_rn(jac_at(J3, i, m), jac_at(J2, m, j)));
            r31[j] = sum;
        }
        for (int j = 0; j < 6; ++j) {
            double sum = 0.0;
            for (int m = 0; m < 2 * n1; ++m) sum = __dadd_rn(sum, __dmul_rn(r31[m], jac_at(J1, m, j)));
            const double t = __dmul_rn(gp[i], sum);
            S[j] = neg ? __dsub_rn(S[j], t) : __dadd_rn(S[j], t);
        }
    }
    const int ia = 2 * order, ib = order != cn - 1 ? 2 * order + 2 : 0;
    const int sa = flip ? 4 : 2, sb = flip ? 2 : 4;
    gAB[ia] = __dadd_rn(gAB[ia], S[sa]);
    gAB[ia + 1] = __dadd_rn(gAB[ia + 1], S[sa + 1]);
    gAB[ib] = __dadd_rn(gAB[ib], S[sb]);
    gAB[ib + 1] = __dadd_rn(gAB[ib + 1], S[sb + 1]);
    return neg ? -res : res;
}

__device__ void giou_row(const float *__restrict__ pf, const float *__restrict__ qf, float *__restrict__ out)
{
    P in[9], A[2 * kUnionMax + 3], B[5];
    bool bad = false;
    for (int t = 0; t < 9; ++t) {
        in[t].x = (double)pf[2 * t]; in[t].y = (double)pf[2 * t + 1];
        bad = bad || !isfinite(in[t].x) || !isfinite(in[t].y);
        A[t] = in[t];
    }
    for (int t = 0; t < 4; ++t) {
        B[t].x = (double)qf[2 * t]; B[t].y = (double)qf[2 * t + 1];
        bad = bad || !isfinite(B[t].x) || !isfinite(B[t].y);
    }
    float g[19];
    for (int t = 0; t < 18; ++t) g[t] = 0.0f;
    if (!bad) {
        // Jarvis_and_index: the hull and, per hull vertex, the first input point equal to it under point_same
        bool closed;
        const int n1 = jarvis<9>(A, 9, closed);
        bad = !closed;
        int to_in[9];
        for (int i = 0; i < n1 && i < 9; ++i) {
            to_in[i] = -1;
            for (int j = 0; j < 9; ++j)
                if (pt_same(A[i], in[j])) { to_in[i] = j; break; }
            bad = bad || to_in[i] < 0;
        }
        bad = bad || n1 > 9;
        if (!bad) {
            // intersectAreaO: both rings counter-clockwise, the gradient written through the ring positions
            double gAB[18], gA[18], gC[18];
            for (int t = 0; t < 18; ++t) { gAB[t] = 0.0; gA[t] = 0.0; gC[t] = 0.0; }
            if (ring_area(A, n1) < 0) reverse_ring(A, n1);
            if (ring_area(B, 4) < 0) reverse_ring(B, 4);
            A[n1] = A[0]; B[4] = B[0];
            double inter = 0.0;
            for (int i = 0; i < n1; ++i)
                for (int j = 0; j < 4; ++j) inter = __dadd_rn(inter, tri_pair_grad(A[i], A[i + 1], B[j], B[j + 1], gAB, i, n1, bad));
            const double sp = area_grad(A, n1, gA);
            if (sp < 0)
                for (int t = 0; t < 2 * n1; ++t) gA[t] = -gA[t];
            const double uni = __dsub_rn(__dadd_rn(fabs(sp), fabs(ring_area(B, 4))), inter);
            const double iou = __ddiv_rn(inter, uni);
            // intersectAreaPoly (convex_giou_kernel.cu:544-616): drop quad points equal to hull points (the scan keeps
            // running over all four slots), hull of the union, gradient through the union vertices that are hull points
            int n2 = 4;
            for (int i = 0; i < n1; ++i)
                for (int j = 0; j < 4; ++j)
                    if (pt_same(A[i], B[j])) {
                        for (int k = j; k < 3; ++k) B[k] = B[k + 1];
                        --n2;
                        break;
                    }
            P U[2 * kUnionMax + 3];
            int nu = n1 + n2;
            for (int i = 0; i < nu; ++i) U[i] = i < n1 ? A[i] : B[i - n1];
            nu = jarvis<kUnionMax>(U, nu, closed);
            bad = bad || !closed;
            double area_u;
            int npred = 0;
            int upos[9], apos[9];
            for (int i = 0; i < nu && !bad; ++i)
                for (int j = 0; j < n1; ++j)
                    if (U[i].x == A[j].x && U[i].y == A[j].y) {
                        if (npred == n1) { bad = true; break; }
                        upos[npred] = i; apos[npred] = j; ++npred;
                        break;
                    }
            if (npred == 0) {
                area_u = fabs(ring_area(U, nu));
            } else {
                double gu[2 * (2 * kUnionMax + 2)];
                area_u = area_grad(U, nu, gu);
                for (int e = 0; e < npred; ++e) { gC[2 * apos[e]] = gu[2 * upos[e]]; gC[2 * apos[e] + 1] = gu[2 * upos[e] + 1]; }
                if (area_u < 0)
                    for (int t = 0; t < 18; ++t) gC[t] = -gC[t];
                area_u = fabs(area_u);
            }
            // combination, convex_giou_kernel.cu:784-796, term by term
            g[18] = (float)__dsub_rn(iou, __ddiv_rn(__dsub_rn(area_u, uni), area_u));
            const double c_ab = __ddiv_rn(__dadd_rn(uni, inter), __dmul_rn(uni, uni));
            const double c_a = __ddiv_rn(iou, uni);
            const double c_d = __ddiv_rn(1.0, area_u);
            const double c_c = __ddiv_rn(__ddiv_rn(uni, area_u), area_u);
            for (int i = 0; i < n1; ++i)
                for (int e = 0; e < 2; ++e) {
                    const int t = 2 * i + e;
                    double v = __dsub_rn(__dmul_rn(c_ab, gAB[t]), __dmul_rn(c_a, gA[t]));
                    v = __dsub_rn(v, __dmul_rn(c_d, __dsub_rn(gAB[t], gA[t])));
                    v = __dsub_rn(v, __dmul_rn(c_c, gC[t]));
                    g[2 * to_in[i] + e] = (float)v;
                }
        }
    }
    if (bad)
        for (int t = 0; t < 19; ++t) g[t] = __int_as_float(0x7fffffff);
    for (int t = 0; t < 19; ++t) out[t] = g[t];
}

__global__ void __launch_bounds__(128)
convex_giou_kernel(const float *__restrict__ pts, const float *__restrict__ quads, int n, float *__restrict__ out)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < (size_t)n; i += (size_t)gridDim.x * blockDim.x)
        giou_row(pts + i * 18, quads + i * 8, out + i * 19);
}

}  // namespace
}  // namespace orp

extern "C" int orp_convex_iou(const float *pts18, int n, const float *quads8, int k, float *out, void *stream)
{
    using namespace orp;
    if (n < 0 || k < 0 || ((size_t)n * k > 0 && (!pts18 || !quads8 || !out))) return fail(ORP_EINVAL, "orp_convex_iou: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const size_t total = (size_t)n * k;
    if (total == 0) return ORP_OK;
    size_t g = (total + 127) / 128;
    if (g > kNumSMs * 32) g = kNumSMs * 32;
    convex_iou_kernel<<<(int)g, 128, 0, static_cast<cudaStream_t>(stream)>>>(pts18, n, quads8, k, out);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_convex_giou(const float *pts18, const float *quads8, int n, float *out19, void *stream)
{
    using namespace orp;
    if (n < 0 || (n > 0 && (!pts18 || !quads8 || !out19))) return fail(ORP_EINVAL, "orp_convex_giou: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    if (n == 0) return ORP_OK;
    size_t g = ((size_t)n + 127) / 128;
    if (g > kNumSMs * 32) g = kNumSMs * 32;
    convex_giou_kernel<<<(int)g, 128, 0, static_cast<cudaStream_t>(stream)>>>(pts18, quads8, n, out19);
    ORP_LAUNCHED();
    return ORP_OK;
}
