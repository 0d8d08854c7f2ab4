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

// Jarvis_and_index (convex_iou_kernel.cu:139-266): gift wrapping from the lowest point, right chain (turn > 0, ties ->
// the farther point) then left chain (turn < 0).  Chains are bounded: the reference loops forever on NaN input.
__device__ int hull9(P *v /* in: 9 points, out: ring */)
{
    constexpr int n = 9;
    P pmax = v[0];
    int imax = 0;
    for (int i = 0; i < n; ++i) {
        if (v[i].y < v[0].y || (v[i].y == v[0].y && v[i].x < v[0].x)) { P t = v[0]; v[0] = v[i]; v[i] = t; }
        if (i == 0) { pmax = v[0]; imax = 0; }
        if (v[i].y > pmax.y || (v[i].y == pmax.y && v[i].x > pmax.x)) { pmax = v[i]; imax = i; }
    }
    if (imax == 0) { imax = 1; pmax = v[1]; }
    int st[2][12], top[2];
    for (int dir = 0; dir < 2; ++dir) {
        int t = 0, k = 0;
        st[dir][0] = 0;
        while (k != imax && t < 10) {
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
        top[dir] = t;
    }
    P out[24];
    const int nh = top[0] + top[1];
    for (int i = 0; i < nh; ++i) out[i] = (i <= top[0]) ? v[st[0][i]] : v[st[1][top[1] - (i - top[0])]];
    for (int i = 0; i < nh; ++i) v[i] = out[i];
    return nh;
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
