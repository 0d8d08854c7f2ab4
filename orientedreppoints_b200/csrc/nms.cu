// nms.cu - rotated / polygon greedy NMS for sm_90a (SURVEY.md section 8 rows a9, a10, a14, a15).
//
// Replaces rnms_cuda (mmdet/ops/nms/src/rnms_kernel.cu:204-265) and _poly_nms
// (DOTA_devkit/poly_nms_gpu/poly_nms_kernel.cu:277-329).  The reference materialises an
// N x N/64 bit matrix (1.25 GB at N = 100k), copies it to the host and scans it there.  Here:
//
//   prep     per box: score key                                                    (1 pass, 4 B/box)
//   sort     CUB radix sorts: by score (rank) and by (segment, xmin) (sweep order)
//   sweep    one warp per box walks its x-interval in the xmin-sorted arrays, lanes test AABBs
//            (coalesced float4), survivors are compacted into a per-warp shared-memory queue and
//            filtered by exact-safe bounds (area bound, projections in both boxes' frames)
//            -> sparse list of CANDIDATE pairs: the only pairs whose IoU can exceed the threshold
//   csr      in-degree scan + scatter: for every box the better-ranked candidates overlapping it
//   resolve  cooperative kernel iterating  keep(i) <=> every better-ranked candidate is suppressed or
//            proven not to suppress i,  suppressed(i) <=> some KEPT candidate has iou > thr  to its
//            (unique) fixed point = greedy NMS.  The polygon clip (fp32 Sutherland-Hodgman in pair-
//            local coordinates; the fp64 reference algorithm inside the error band) is evaluated LAZILY,
//            only for pairs (undecided box, kept candidate): a suppressed box never suppresses, so the
//            IoU of every pair whose better box ends up suppressed is never needed - on a dense tile
//            that removes ~97 % of the clips a full suppression graph would take
//   select   CUB flagged select into the caller's int64 buffer, count stays on the device
//
// Nothing touches the host; no N^2 memory.
#include <cooperative_groups.h>
#include <cub/cub.cuh>
#include <vector>

#include "common.cuh"
#include "geom.cuh"

namespace cg = cooperative_groups;

namespace orp {

struct NmsCounters {
    unsigned long long pairs_swept, pairs_aabb, pairs_clipped, pairs_fp64, edges, suppressing;
    int overflow;
    int rounds;
};

static thread_local int g_last_n;
static thread_local cudaEvent_t g_ev[2] = {nullptr, nullptr};
static thread_local NmsCounters *g_stats_pinned = nullptr;
static thread_local orp_rnms_plan g_last_plan;
static thread_local bool g_have_plan = false;

// per-box `area` value of a quadrilateral whose fp64 signed area (ring_area<double>, the area of the fp64 decision) is
// exactly zero; like every negative value it keeps the box out of the fp32 bounds and the fast path
constexpr float kZeroArea = -2.0f;

// ---------------------------------------------------------------------------------------------
// prep: keys for the rank sort
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
nms_prep_kernel(const float *__restrict__ dets, int n, uint32_t *__restrict__ score_key, int32_t *__restrict__ iota)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *d = dets + (size_t)i * 9;
    // -0.0 and +0.0 are equal scores: one key, so that the tie rule (lower index first) holds between them
    const float sc = (__float_as_uint(d[8]) << 1) == 0u ? 0.0f : d[8];
    score_key[i] = ~orderable(sc);                         // ascending key == descending score
    iota[i] = i;
}

__global__ void __launch_bounds__(256)
nms_rank_kernel(const int32_t *__restrict__ order, int n, int32_t *__restrict__ rank)
{
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n) rank[order[r]] = r;
}

// ---------------------------------------------------------------------------------------------
// EXACT64 candidate search: per-box arrays (by ORIGINAL index) + "registrations" for the sweep
// ---------------------------------------------------------------------------------------------
// Global facts the registration needs, gathered without a host round trip.
struct NmsGlobal {
    unsigned int ymin_key;        // orderable(min AABB ymin) over finite boxes
    unsigned int maxh_bits;       // float bits of the largest AABB height (non-negative: bit order == value order)
    unsigned int maxabs_bits;     // float bits of the largest |coordinate|
    double sumh;                  // sum of AABB heights
    unsigned int count;           // finite boxes
};

__device__ __forceinline__ float from_orderable(uint32_t k)
{
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

// per box: vertices, AABB, area sign (convexity); block-reduced global statistics
__global__ void __launch_bounds__(256)
nms_boxes_kernel(const float *__restrict__ dets, int n, float4 *__restrict__ baabb, float4 *__restrict__ v01,
                 float4 *__restrict__ v23, float *__restrict__ area, NmsGlobal *__restrict__ G)
{
    __shared__ unsigned int s_ymin, s_maxh, s_cnt, s_maxabs;
    __shared__ float s_sum;
    if (threadIdx.x == 0) { s_ymin = 0xFFFFFFFFu; s_maxh = 0u; s_cnt = 0u; s_sum = 0.f; s_maxabs = 0u; }
    __syncthreads();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float *d = dets + (size_t)i * 9;
        float c[8];
        bool finite = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) { c[k] = d[k]; finite = finite && isfinite(c[k]); }
        const float xmin = fminf(fminf(c[0], c[2]), fminf(c[4], c[6])), xmax = fmaxf(fmaxf(c[0], c[2]), fmaxf(c[4], c[6]));
        const float ymin = fminf(fminf(c[1], c[3]), fminf(c[5], c[7])), ymax = fmaxf(fmaxf(c[1], c[3]), fmaxf(c[5], c[7]));
        baabb[i] = make_float4(xmin, ymin, xmax, ymax);
        v01[i] = make_float4(c[0], c[1], c[2], c[3]);
        v23[i] = make_float4(c[4], c[5], c[6], c[7]);
        // area about the box's own first vertex (small coordinates -> accurate); negative marks "not a convex
        // quadrilateral": such boxes are never pruned by the area bound and are always decided by the fp64 reference
        // algorithm (which accepts arbitrary quadrilaterals); NaN area (non-finite box) never takes part
        const float ux = c[2] - c[0], uy = c[3] - c[1], vx = c[4] - c[0], vy = c[5] - c[1], wx = c[6] - c[0], wy = c[7] - c[1];
        area[i] = quad_is_convex(c) ? 0.5f * fabsf((ux * vy - uy * vx) + (vx * wy - vy * wx)) : -1.0f;
        if (finite) {
            Pt<double> P[5];
#pragma unroll
            for (int k = 0; k < 4; ++k) { P[k].x = (double)c[2 * k]; P[k].y = (double)c[2 * k + 1]; }
            if (ring_area(P, 4) == 0.0) area[i] = kZeroArea;
        }
        if (finite) {
            atomicMin(&s_ymin, orderable(ymin));
            atomicMax(&s_maxh, __float_as_uint(ymax - ymin));
            atomicMax(&s_maxabs, __float_as_uint(fmaxf(fmaxf(fabsf(xmin), fabsf(xmax)), fmaxf(fabsf(ymin), fabsf(ymax)))));
            atomicAdd(&s_sum, ymax - ymin);
            atomicAdd(&s_cnt, 1u);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt) {
        atomicMin(&G->ymin_key, s_ymin);
        atomicMax(&G->maxh_bits, s_maxh);
        atomicMax(&G->maxabs_bits, s_maxabs);
        atomicAdd(&G->sumh, (double)s_sum);
        atomicAdd(&G->count, s_cnt);
    }
}

// Strip geometry shared by registration and sweep (identical arithmetic on both sides): strips of height s along y,
// s >= max AABB height / 3 so that a box overlaps at most 4 strips; R == 1 disables the strips (one strip holds everything).
struct Strips {
    float y0, s;
    __device__ __forceinline__ int of(float y) const { return (int)floorf((y - y0) / s); }
};
__device__ __forceinline__ Strips make_strips(const NmsGlobal *G, int R)
{
    Strips S;
    S.y0 = from_orderable(G->ymin_key);
    if (R == 1 || G->count == 0) { S.s = 3.0e38f; return S; }
    const float maxh = __uint_as_float(G->maxh_bits), meanh = (float)(G->sumh / (double)G->count);
    S.s = fmaxf(fmaxf(1.5f * meanh, maxh * (1.0001f / 3.0f)), 1e-6f);
    return S;
}

// R registration slots per box: one per strip its AABB overlaps (key = segment : strip : xmin), the rest padded with
// all-ones keys that sort to the end.  A pair is examined only in the strip that holds max(ymin_i, ymin_j), so it is
// seen exactly once although both boxes may be registered in several common strips.
__global__ void __launch_bounds__(256)
nms_regs_kernel(const float4 *__restrict__ baabb, const int32_t *__restrict__ segments, int n, int R,
                const NmsGlobal *__restrict__ G, uint64_t *__restrict__ keys, int32_t *__restrict__ vals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 b = baabb[i];
    const bool finite = isfinite(b.x) && isfinite(b.y) && isfinite(b.z) && isfinite(b.w);
    const Strips S = make_strips(G, R);
    int t0 = 0, t1 = -1;
    if (finite) { t0 = S.of(b.y); t1 = S.of(b.w); if (R == 1) t1 = t0 = 0; if (t1 - t0 > R - 1) t1 = t0 + R - 1; }
    if (R == 1) {
        // no strips: the whole upper word is the segment id (31 bits)
        const uint64_t seg = segments ? (uint64_t)((uint32_t)segments[i] & 0x7FFFFFFFu) : 0ull;
        keys[i] = finite ? ((seg << 32) | orderable(b.x)) : ~0ull;
        vals[i] = i;
        return;
    }
    const uint64_t seg = segments ? (uint64_t)((uint32_t)segments[i] & 0x7FFFu) : 0ull;
    for (int k = 0; k < R; ++k) {
        const int t = t0 + k;
        keys[(size_t)i * R + k] = (t <= t1) ? ((seg << 48) | ((uint64_t)(uint32_t)(t & 0xFFFF) << 32) | orderable(b.x)) : ~0ull;
        vals[(size_t)i * R + k] = i;
    }
}

// sorted registrations -> the arrays the sweep streams: AABB and (group = segment : strip, box id, area, rank)
__global__ void __launch_bounds__(256)
nms_slots_kernel(const uint64_t *__restrict__ keys, const int32_t *__restrict__ vals, const float4 *__restrict__ baabb,
                 const float *__restrict__ area, const int32_t *__restrict__ rank, int m,
                 float4 *__restrict__ aabb_s, int4 *__restrict__ meta_s, int32_t *__restrict__ nvalid)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= m) return;
    const uint64_t k = keys[s];
    const bool valid = (k != ~0ull);
    const int i = vals[s];
    aabb_s[s] = baabb[i];
    // everything the sweep needs about the slot's box next to its AABB: no dependent gathers while walking
    meta_s[s] = make_int4((int32_t)(k >> 32), i, __float_as_int(area[i]), rank[i]);
    const bool prev_valid = (s == 0) ? true : (keys[s - 1] != ~0ull);
    if (!valid && prev_valid) *nvalid = s;                   // first padding slot = number of registrations
    if (valid && s == m - 1) *nvalid = m;
}

// Zero-area lists (ORP_UNION_GUARD / ORP_UNION_NAN_SUPPRESSES_ALL): these conventions compare every pair, and for two
// (near-)degenerate boxes the fp64 IoU is a ratio of rounding residues (NaN, -1 or anything), whatever their distance.
// Such boxes are compared with each other explicitly: every one gets the segment's worse-ranked ones as implicit
// candidates.  Degenerate = |fp64 signed area| <= 2^-36 S^2, S = the largest |coordinate| of the set: the shoelace sum of
// a collinear ring rounds to at most a few 2^-53 S^2, and a fan residue (<= ~2^-47 S^2) over a box above the bound stays
// far below any threshold, so pairs with one box above it need no explicit comparison.  Sort key per rank: the segment of
// a finite degenerate box, `none` for every other box; a stable sort keeps rank order inside a segment.
__global__ void __launch_bounds__(256)
nms_zero_keys_kernel(const int32_t *__restrict__ order, const int32_t *__restrict__ segments, const float4 *__restrict__ v01,
                     const float4 *__restrict__ v23, const NmsGlobal *__restrict__ G, int n, uint32_t none, float *__restrict__ area,
                     uint32_t *__restrict__ keys)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int i = order[r];
    const float4 a = v01[i], b = v23[i];
    Pt<double> P[5];
    P[0].x = a.x; P[0].y = a.y; P[1].x = a.z; P[1].y = a.w; P[2].x = b.x; P[2].y = b.y; P[3].x = b.z; P[3].y = b.w;
    const double S = fmax(1.0, (double)__uint_as_float(G->maxabs_bits));
    const bool deg = fabs(ring_area(P, 4)) <= ldexp(S * S, -36);      // NaN (non-finite box): false
    if (deg) area[i] = kZeroArea;
    keys[r] = deg ? (segments ? ((uint32_t)segments[i] & 0x7FFFFFFFu) : 0u) : none;
}

// sorted zero-area list -> per zero-area box: its list position, the end of its segment's run and how many better-ranked
// zero-area boxes of its segment precede it (its extra pending count)
__global__ void __launch_bounds__(256)
nms_zero_list_kernel(const uint32_t *__restrict__ keys, const int32_t *__restrict__ zlist, int n, uint32_t none,
                     int32_t *__restrict__ zpos, int32_t *__restrict__ zhi, int32_t *__restrict__ zbetter)
{
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t k = keys[p];
    if (k == none) return;
    int a = 0, b = p;
    while (a < b) { const int mid = (a + b) >> 1; if (keys[mid] < k) a = mid + 1; else b = mid; }
    int c = p + 1, d = n;
    while (c < d) { const int mid = (c + d) >> 1; if (keys[mid] <= k) c = mid + 1; else d = mid; }
    const int box = zlist[p];
    zpos[box] = p;
    zhi[box] = c;
    zbetter[box] = p - a;
}

// after the sweep (every attempt resets `pending`): a zero-area box also waits for the better zero-area boxes of its segment
__global__ void __launch_bounds__(256)
nms_zero_pending_kernel(const int32_t *__restrict__ zpos, const int32_t *__restrict__ zbetter, int n, int32_t *__restrict__ pending)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && zpos[i] >= 0) pending[i] += zbetter[i];
}

// COMPAT32: the tile kernel's inputs (vertices, segment) in `perm` order
__global__ void __launch_bounds__(256)
nms_gather_kernel(const float *__restrict__ dets, const int32_t *__restrict__ segments, const int32_t *__restrict__ perm,
                  int n, float4 *__restrict__ v01, float4 *__restrict__ v23, int32_t *__restrict__ sg)
{
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int i = perm[s];
    const float *d = dets + (size_t)i * 9;
    v01[s] = make_float4(d[0], d[1], d[2], d[3]);
    v23[s] = make_float4(d[4], d[5], d[6], d[7]);
    sg[s] = segments ? segments[i] : 0;
}

// ---------------------------------------------------------------------------------------------
// pair decision
// ---------------------------------------------------------------------------------------------
struct Quad { float c[8]; };

// The reference's fp64 arithmetic for one pair, evaluated by a whole warp: its 16 (edge of A, edge of B) fan terms are
// independent, so lane l < 16 computes term (l / 4, l % 4) and the terms are then added in the reference's order
// (polyiou.cpp:122-131: i outer, j inner) - same bits as the serial loop at 1/16 of its latency.  Every lane of the
// warp must call it with the same quads.
__device__ __noinline__ bool decide_fp64_warp(const Quad &A, const Quad &B, double thr, int union_mode, int lane)
{
    using R = Rn<double>;
    Pt<double> P[6], Q[6];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        P[i].x = (double)A.c[2 * i]; P[i].y = (double)A.c[2 * i + 1];
        Q[i].x = (double)B.c[2 * i]; Q[i].y = (double)B.c[2 * i + 1];
    }
    if (ring_area(P, 4) < 0) { Pt<double> t = P[0]; P[0] = P[3]; P[3] = t; t = P[1]; P[1] = P[2]; P[2] = t; }
    if (ring_area(Q, 4) < 0) { Pt<double> t = Q[0]; Q[0] = Q[3]; Q[3] = t; t = Q[1]; Q[1] = Q[2]; Q[2] = t; }
    P[4] = P[0]; Q[4] = Q[0];
    const int i = (lane >> 2) & 3, j = lane & 3;
    const double v = fan_pair(P[i], P[i + 1], Q[j], Q[j + 1]);
    PairRes<double> r;
    r.inter = 0;
    for (int k = 0; k < 16; ++k) r.inter = R::add(r.inter, __shfl_sync(0xffffffffu, v, k));
    const double ap = ring_area(P, 4), aq = ring_area(Q, 4);
    r.area_p = ap < 0 ? -ap : ap;
    r.area_q = aq < 0 ? -aq : aq;
    const double iou = iou_from<double>(r, union_mode);
    return suppresses<double>(iou, thr, union_mode);
}

// 1 / 0: the reference's fp64 IoU of (A, B) certainly suppresses / does not suppress at thr (fp32 clip with an error band);
// -1: inside the band, or not a pair of convex quadrilaterals -> decide_fp64_warp
__device__ __forceinline__ int decide_fast(const Quad &A, const Quad &B, const float4 &ba, const float4 &bb, bool both_convex,
                                           double thr, float *scratch)
{
    if (!both_convex) return -1;
    const float ox = 0.5f * (fmaxf(ba.x, bb.x) + fminf(ba.z, bb.z));
    const float oy = 0.5f * (fmaxf(ba.y, bb.y) + fminf(ba.w, bb.w));
    float a[8], b[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        a[2 * k] = A.c[2 * k] - ox; a[2 * k + 1] = A.c[2 * k + 1] - oy;
        b[2 * k] = B.c[2 * k] - ox; b[2 * k + 1] = B.c[2 * k + 1] - oy;
    }
    FastRes r = fast_quad_pair_s<1>(a, b, scratch);
    const float t = (float)thr;
    const float margin = r.inter * (1.f + t) - t * (r.area_a + r.area_b);
    const float band = 4.f * r.err + 1e-6f * (r.area_a + r.area_b);
    if (fabsf(margin) > band) return margin > 0.f ? 1 : 0;
    return -1;
}

struct SweepParams {
    const float4 *aabb_s;                      // per registration slot (sweep order)
    const int4 *meta_s;                        // (group, box id, area bits, rank)
    const float4 *v01, *v23;                   // per box (original index)
    const int32_t *nvalid;
    const NmsGlobal *G;
    int R;
    int2 *edges;                               // (better-ranked box, worse-ranked box)
    int32_t *outdeg;                           // per better box: how many worse boxes list it as a candidate
    int32_t *pending;                          // per worse box: candidates not resolved yet
    unsigned long long edge_cap;
    NmsCounters *ctr;
    double thr;
    int union_mode;
};

constexpr int kSweepWarps = 8;

// Exact-safe rejection in the frame of quad P (u = first edge, v = u rotated by 90 degrees): the
// intersection of P and Q lies inside the rectangle [overlap of the two projections on u] x [overlap on v],
// so  inter <= ou * ov / |u|^2.  No overlap on either axis = a separating axis = empty intersection.
// Returns true when  iou <= thr  is certain (with a 0.2 % margin against fp32 rounding).
__device__ __forceinline__ bool frame_prune(const float *p, const float *q, float kthr_sum)
{
    const float ux = p[2] - p[0], uy = p[3] - p[1];
    const float l2 = ux * ux + uy * uy;
    if (!(l2 > 0.f)) return false;
    float pu0 = 0.f, pu1 = 0.f, pv0 = 0.f, pv1 = 0.f;            // P's own vertex 0 projects to (0, 0)
    float qu0 = 3.4e38f, qu1 = -3.4e38f, qv0 = 3.4e38f, qv1 = -3.4e38f;
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        const float dx = p[2 * k] - p[0], dy = p[2 * k + 1] - p[1];
        const float a = dx * ux + dy * uy, c = dy * ux - dx * uy;
        pu0 = fminf(pu0, a); pu1 = fmaxf(pu1, a); pv0 = fminf(pv0, c); pv1 = fmaxf(pv1, c);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float dx = q[2 * k] - p[0], dy = q[2 * k + 1] - p[1];
        const float a = dx * ux + dy * uy, c = dy * ux - dx * uy;
        qu0 = fminf(qu0, a); qu1 = fmaxf(qu1, a); qv0 = fminf(qv0, c); qv1 = fmaxf(qv1, c);
    }
    const float ou = fminf(pu1, qu1) - fmaxf(pu0, qu0), ov = fminf(pv1, qv1) - fmaxf(pv0, qv0);
    if (ou <= 0.f || ov <= 0.f) return true;                     // separating axis
    return (ou * ov) < 0.998f * kthr_sum * l2;                   // inter <= ou*ov/l2 < thr/(1+thr) * (A+B)
}

// One warp per registration slot i: walk the slots after it while they stay in the same (segment, strip) group and
// start left of i's right edge; lanes test AABBs (coalesced float4 reads of the sorted array), survivors of the area bound
// are compacted into a per-warp shared-memory queue, filtered by the projection bounds in both boxes' frames, and emitted
// as candidate pairs (better-ranked box, worse-ranked box) by ORIGINAL index.
__global__ void __launch_bounds__(kSweepWarps * 32, 4)
nms_sweep_kernel(SweepParams P)
{
    __shared__ int32_t q1[kSweepWarps][64];    // AABB + area-bound survivors: box id,
    __shared__ int32_t q1r[kSweepWarps][64];   //   rank,
    __shared__ float q1a[kSweepWarps][64];     //   area
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nv = *P.nvalid;
    const int nwarps = gridDim.x * kSweepWarps;
    unsigned long long c_swept = 0, c_aabb = 0;
    const float thrf = (float)P.thr;
    const float kthr = thrf / (1.f + thrf);
    const unsigned lt = (1u << lane) - 1u;
    const Strips S = make_strips(P.G, P.R);

    for (int i = blockIdx.x * kSweepWarps + wib; i < nv; i += nwarps) {
        const float4 ba = P.aabb_s[i];
        const int4 mi = P.meta_s[i];
        const int grp_i = mi.x;
        const int strip_i = grp_i & 0xFFFF;
        const int bi = mi.y;
        const int rk_i = mi.w;
        const float area_i = __int_as_float(mi.z);
        float A[8];
        {
            const float4 t0 = P.v01[bi], t1 = P.v23[bi];
            A[0] = t0.x; A[1] = t0.y; A[2] = t0.z; A[3] = t0.w; A[4] = t1.x; A[5] = t1.y; A[6] = t1.z; A[7] = t1.w;
        }
        int n1 = 0;
        bool more = true;
        for (int base = i + 1;; base += 32) {
            // ---- stage 0: walk the x-interval, AABB test + strip ownership + area bound -> q1
            bool hit = false;
            const int j = base + lane;
            int4 mj = make_int4(0, 0, 0, 0);
            if (more) {
                bool cont = false;
                if (j < nv) {
                    const float4 bb = P.aabb_s[j];
                    mj = P.meta_s[j];
                    cont = (mj.x == grp_i) && (bb.x <= ba.z);
                    if (cont) {
                        ++c_swept;
                        // the AABB intersection has positive area (py_cpu_nms_poly_fast's `hbb_ovr > 0`): a box with a
                        // zero-width or zero-height AABB has zero area and pairs with nothing here (bb.x >= ba.x: sweep order)
                        hit = (bb.x < ba.z) && (bb.z > bb.x) && (bb.y < ba.w) && (bb.w > ba.y) && (ba.w > ba.y) && (bb.w > bb.y);
                        // the pair belongs to the strip holding the top of the AABB intersection
                        if (hit && P.R > 1) hit = ((S.of(fmaxf(ba.y, bb.y)) & 0xFFFF) == strip_i);
                        if (hit) {
                            ++c_aabb;
                            // exact-safe area bound: inter <= min(area_i, area_j, |AABB_i ^ AABB_j|)
                            const float iw = fminf(ba.z, bb.z) - fmaxf(ba.x, bb.x);
                            const float ih = fminf(ba.w, bb.w) - fmaxf(ba.y, bb.y);
                            const float area_j = __int_as_float(mj.z);
                            const float imax = fminf(fminf(area_i, area_j), iw * ih);
                            if (imax * (1.f + thrf) < 0.999f * thrf * (area_i + area_j) && imax > 0.f) hit = false;
                        }
                    }
                }
                more = __all_sync(0xffffffffu, cont);
            }
            const unsigned hm = __ballot_sync(0xffffffffu, hit);
            if (hit) {
                const int at = n1 + __popc(hm & lt);
                q1[wib][at] = mj.y; q1r[wib][at] = mj.w; q1a[wib][at] = __int_as_float(mj.z);
            }
            n1 += __popc(hm);
            __syncwarp();
            // ---- stage 1: projection bounds in both frames -> candidate pairs
            while (n1 >= 32 || (!more && n1 > 0)) {
                const int take = n1 < 32 ? n1 : 32;
                bool pass = false;
                int bj = 0, rk_j = 0;
                if (lane < take) {
                    bj = q1[wib][n1 - take + lane];
                    rk_j = q1r[wib][n1 - take + lane];
                    const float area_j = q1a[wib][n1 - take + lane];
                    pass = true;
                    if (area_i >= 0.f && area_j >= 0.f) {             // both convex: bounds are valid
                        float b[8];
                        const float4 t0 = P.v01[bj], t1 = P.v23[bj];
                        b[0] = t0.x; b[1] = t0.y; b[2] = t0.z; b[3] = t0.w; b[4] = t1.x; b[5] = t1.y; b[6] = t1.z; b[7] = t1.w;
                        const float ks = kthr * (area_i + area_j);
                        if (ks > 0.f && (frame_prune(A, b, ks) || frame_prune(b, A, ks))) pass = false;
                    }
                }
                n1 -= take;
                const unsigned pm = __ballot_sync(0xffffffffu, pass);
                if (pm) {
                    unsigned long long basep = 0;
                    if (lane == 0) basep = atomicAdd(&P.ctr->edges, (unsigned long long)__popc(pm));
                    basep = __shfl_sync(0xffffffffu, basep, 0);
                    if (pass) {
                        const unsigned long long pos = basep + __popc(pm & lt);
                        const bool i_worse = rk_i > rk_j;
                        const int lo = i_worse ? bi : bj, hi = i_worse ? bj : bi;
                        if (pos < P.edge_cap) {
                            P.edges[pos] = make_int2(hi, lo);
                            atomicAdd(&P.outdeg[hi], 1);
                            atomicAdd(&P.pending[lo], 1);
                        } else {
                            P.ctr->overflow = 1;
                        }
                    }
                }
                __syncwarp();
            }
            if (!more) break;
        }
    }
    // one atomic per warp per counter
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        c_swept += __shfl_down_sync(0xffffffffu, c_swept, o);
        c_aabb += __shfl_down_sync(0xffffffffu, c_aabb, o);
    }
    if (lane == 0) {
        atomicAdd(&P.ctr->pairs_swept, c_swept);
        atomicAdd(&P.ctr->pairs_aabb, c_aabb);
    }
}

// ---------------------------------------------------------------------------------------------
// COMPAT32: every pair of the upper triangle with the reference's fp32 arithmetic
// (rnms_kernel.cu:149-201: 64 x 64 tiles, column boxes staged in shared memory)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(64)
nms_compat_tiles_kernel(const float4 *__restrict__ v01, const float4 *__restrict__ v23,
                        const int32_t *__restrict__ sg, int n, float thr, int union_mode,
                        int2 *edges, int32_t *indeg, unsigned long long edge_cap, NmsCounters *ctr)
{
    // linear upper-triangle tile index -> (rb, cb), cb >= rb
    const int nb = (n + 63) / 64;
    long long t = blockIdx.x;
    int rb = 0;
    {
        // row rb has (nb - rb) tiles; solve by a short loop on one thread, broadcast via smem
        __shared__ int s_rb, s_cb;
        if (threadIdx.x == 0) {
            long long rem = t;
            int r = 0;
            // closed form start then fix up
            double nbd = (double)nb;
            r = (int)floor(((2.0 * nbd + 1.0) - sqrt((2.0 * nbd + 1.0) * (2.0 * nbd + 1.0) - 8.0 * (double)t)) * 0.5);
            if (r < 0) r = 0;
            if (r >= nb) r = nb - 1;
            auto start = [&](int rr) { return (long long)rr * nb - (long long)rr * (rr - 1) / 2; };
            while (r > 0 && start(r) > t) --r;
            while (r + 1 < nb && start(r + 1) <= t) ++r;
            rem = t - start(r);
            s_rb = r;
            s_cb = r + (int)rem;
        }
        __syncthreads();
        rb = s_rb;
        t = s_cb;
    }
    const int cb = (int)t;
    __shared__ float col[64][8];
    __shared__ int colseg[64];
    const int cj = cb * 64 + threadIdx.x;
    if (cj < n) {
        float4 a = v01[cj], b = v23[cj];
        col[threadIdx.x][0] = a.x; col[threadIdx.x][1] = a.y; col[threadIdx.x][2] = a.z; col[threadIdx.x][3] = a.w;
        col[threadIdx.x][4] = b.x; col[threadIdx.x][5] = b.y; col[threadIdx.x][6] = b.z; col[threadIdx.x][7] = b.w;
        colseg[threadIdx.x] = sg[cj];
    }
    __syncthreads();
    const int ri = rb * 64 + threadIdx.x;
    if (ri >= n) return;
    float p[8];
    {
        float4 a = v01[ri], b = v23[ri];
        p[0] = a.x; p[1] = a.y; p[2] = a.z; p[3] = a.w; p[4] = b.x; p[5] = b.y; p[6] = b.z; p[7] = b.w;
    }
    const int seg_i = sg[ri];
    const int ncol = min(64, n - cb * 64);
    const int start = (rb == cb) ? threadIdx.x + 1 : 0;
    unsigned long long clipped = 0;
    for (int c = start; c < ncol; ++c) {
        if (colseg[c] != seg_i) continue;
        float q[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) q[k] = col[c][k];
        PairRes<float> r = ref_quad_pair<float>(p, q);
        float iou = iou_from<float>(r, union_mode);
        ++clipped;
        if (suppresses<float>(iou, thr, union_mode)) {
            unsigned long long pos = atomicAdd(&ctr->edges, 1ull);
            if (pos < edge_cap) {
                const int lo = cb * 64 + c, hi = ri;   // arrays are in rank order: row is better
                edges[pos] = make_int2(lo, hi);
                atomicAdd(&indeg[lo], 1);
            } else {
                ctr->overflow = 1;
            }
        }
    }
    atomicAdd(&ctr->pairs_clipped, clipped);
}

// ---------------------------------------------------------------------------------------------
// CSR scatter + greedy resolution
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
nms_scatter_kernel(const int2 *__restrict__ edges, const NmsCounters *__restrict__ ctr,
                   unsigned long long edge_cap, const int32_t *__restrict__ offs,
                   int32_t *__restrict__ cursor, int32_t *__restrict__ adj)
{
    unsigned long long ne = ctr->edges < edge_cap ? ctr->edges : edge_cap;
    for (unsigned long long e = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; e < ne;
         e += (unsigned long long)gridDim.x * blockDim.x) {
        int2 ed = edges[e];
        int pos = offs[ed.x] + atomicAdd(&cursor[ed.x], 1);
        adj[pos] = ed.y;
    }
}

// status by rank: 0 undecided, 1 kept, 2 suppressed
__global__ void __launch_bounds__(256)
nms_resolve_kernel(const int32_t *__restrict__ offs, const int32_t *__restrict__ adj, int n,
                   volatile uint8_t *status, int *changed /* [2] */, NmsCounters *ctr)
{
    cg::grid_group grid = cg::this_grid();
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int nth = gridDim.x * blockDim.x;
    int round = 0;
    while (true) {
        int *flag = &changed[round & 1];
        int local = 0;
        for (int r = tid; r < n; r += nth) {
            if (status[r] != 0) continue;
            const int b = offs[r], e = offs[r + 1];
            bool any_keep = false, all_supp = true;
            for (int k = b; k < e; ++k) {
                const uint8_t s = status[adj[k]];
                if (s == 1) { any_keep = true; break; }
                if (s == 0) all_supp = false;
            }
            if (any_keep) { status[r] = 2; local = 1; }
            else if (all_supp) { status[r] = 1; local = 1; }
        }
        if (local) *flag = 1;
        __threadfence();
        grid.sync();
        const int any = *(volatile int *)flag;
        if (tid == 0) changed[(round + 1) & 1] = 0;
        ++round;
        grid.sync();
        if (!any) break;
    }
    if (tid == 0) ctr->rounds = round;
}

// Lazy variant (EXACT64 mode).  The sweep leaves CANDIDATE pairs; a candidate is clipped only when its better-ranked box is
// known to be kept and the worse one is still undecided, and nothing is ever scanned twice: the graph is stored by the
// BETTER box (out lists of worse boxes) and every box carries `pending` = candidates not resolved yet.  Decisions travel
// along the out lists of the boxes decided in the previous round (two frontiers):
//   phase 1 (warp per frontier box): a newly KEPT box queues (worse box, itself) for clipping, for every undecided worse box;
//            a newly SUPPRESSED box resolves itself in its worse boxes (pending -= 1);
//   phase 2 (thread per queued pair): decide the pair exactly; "suppresses" -> the worse box is suppressed (first writer joins
//            the suppressed frontier), otherwise the pair is resolved (pending -= 1).
// pending reaching 0 means every better candidate is suppressed or proven harmless: the box is kept (exactly one decrement
// sees 1 -> 0, and a box with a suppressing pair never gets there because that pair is never resolved).  Statuses only move
// undecided -> final and each decision uses final statuses only, so the fixed point is the greedy result whatever the order.
// Total work is O(candidates) + the clips, instead of a rescan of every live list per round.
struct LazyParams {
    const int32_t *offs;                       // out lists: offs[j] .. offs[j] + deg[j]
    const int32_t *adj;
    const int32_t *deg;
    int n;
    int32_t *status;                           // by original index: 0 undecided, 1 kept, 2 suppressed
    int32_t *pending;
    NmsCounters *ctr;
    unsigned int *counts;                      // [0..1] kept frontier fill by round parity, [2..3] suppressed frontier, [4..5] queue
    int32_t *fkept, *fsup;                     // [2][n] each
    int2 *queue;                               // (worse box, better box); capacity = number of candidates
    const float4 *aabb, *v01, *v23;
    const float *area;
    double thr;
    int union_mode;
    const int32_t *zlist, *zpos, *zhi;         // zero-area lists (NULL: none): a zero-area box j also has the worse zero-area
                                               // boxes zlist[zpos[j] + 1 .. zhi[j]) of its segment as candidates
};

__global__ void __launch_bounds__(256, 4)
nms_resolve_lazy_kernel(LazyParams P)
{
    cg::grid_group grid = cg::this_grid();
    float scratch[40];
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int nth = gridDim.x * blockDim.x;
    const int lane = threadIdx.x & 31, gwarp = tid >> 5, nwarps = nth >> 5;
    const unsigned lt = (1u << lane) - 1u;
    unsigned long long c_clip = 0, c_64 = 0, c_sup = 0;
    // boxes nobody better overlaps are kept outright: the first frontier
    for (int r0 = blockIdx.x * blockDim.x; r0 < P.n; r0 += nth) {
        const int r = r0 + threadIdx.x;
        const bool k = r < P.n && P.pending[r] == 0;
        const unsigned m = __ballot_sync(0xffffffffu, k);
        if (m) {
            unsigned int base = 0;
            if (lane == 0) base = atomicAdd(&P.counts[0], (unsigned int)__popc(m));
            base = __shfl_sync(0xffffffffu, base, 0);
            if (k) { P.status[r] = 1; P.fkept[base + __popc(m & lt)] = r; }
        }
    }
    __threadfence();
    grid.sync();
    int round = 0;
    while (true) {
        const int cur = round & 1, nxt = cur ^ 1;
        const unsigned int nk = *(volatile unsigned int *)&P.counts[cur];
        const unsigned int ns = *(volatile unsigned int *)&P.counts[2 + cur];
        if (nk == 0 && ns == 0) break;
        const int32_t *fk = P.fkept + (size_t)cur * P.n, *fs = P.fsup + (size_t)cur * P.n;
        int32_t *fk_next = P.fkept + (size_t)nxt * P.n, *fs_next = P.fsup + (size_t)nxt * P.n;
        unsigned int *qc = &P.counts[4 + cur];
        // ---- phase 1
        for (unsigned int w = gwarp; w < nk + ns; w += nwarps) {
            const bool kept = w < nk;
            const int j = kept ? fk[w] : fs[w - nk];
            // the out list, then (zero-area box) the rest of its segment's zero-area list
            for (int pass = 0; pass < 2; ++pass) {
                const int32_t *list = pass == 0 ? P.adj : P.zlist;
                int b = 0, e = 0;
                if (pass == 0) { b = P.offs[j]; e = b + P.deg[j]; }
                else if (P.zpos && P.zpos[j] >= 0) { b = P.zpos[j] + 1; e = P.zhi[j]; }
                // four chunks of the list in flight per warp: the walk is a chain of dependent loads (entry -> status -> atomic)
                for (int k0 = b; k0 < e; k0 += 128) {
                    int r[4];
                    bool act[4];
    #pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int k = k0 + 32 * u + lane;
                        r[u] = k < e ? list[k] : -1;
                    }
    #pragma unroll
                    for (int u = 0; u < 4; ++u) act[u] = r[u] >= 0 && *(volatile int32_t *)&P.status[r[u]] == 0;
                    if (kept) {
    #pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const unsigned m = __ballot_sync(0xffffffffu, act[u]);
                            if (m) {
                                unsigned int base = 0;
                                if (lane == 0) base = atomicAdd(qc, (unsigned int)__popc(m));
                                base = __shfl_sync(0xffffffffu, base, 0);
                                if (act[u]) P.queue[base + __popc(m & lt)] = make_int2(r[u], j);
                            }
                        }
                    } else {
    #pragma unroll
                        for (int u = 0; u < 4; ++u)
                            if (act[u] && atomicSub(&P.pending[r[u]], 1) == 1) {
                                P.status[r[u]] = 1;
                                fk_next[atomicAdd(&P.counts[nxt], 1u)] = r[u];
                            }
                    }
                }
            }
        }
        __threadfence();
        grid.sync();
        const unsigned int nq = *(volatile unsigned int *)qc;
        if (tid == 0) { P.counts[cur] = 0; P.counts[2 + cur] = 0; P.counts[4 + nxt] = 0; }
        // ---- phase 2 (the loop bound is warp-uniform: pairs the fp32 clip cannot decide are finished by the whole warp)
        for (unsigned int q0 = (unsigned int)(tid - lane); q0 < nq; q0 += nth) {
            const unsigned int q = q0 + lane;
            int r = -1, j = -1, res = 0;
            bool valid = q < nq;
            Quad A, B;
            if (valid) {
                const int2 e = P.queue[q];
                r = e.x; j = e.y;
                valid = *(volatile int32_t *)&P.status[r] == 0;    // else another pair of this round already suppressed it
            }
            if (valid) {
                const float4 t0 = P.v01[r], t1 = P.v23[r];
                A.c[0] = t0.x; A.c[1] = t0.y; A.c[2] = t0.z; A.c[3] = t0.w; A.c[4] = t1.x; A.c[5] = t1.y; A.c[6] = t1.z; A.c[7] = t1.w;
                const float4 u0 = P.v01[j], u1 = P.v23[j];
                B.c[0] = u0.x; B.c[1] = u0.y; B.c[2] = u0.z; B.c[3] = u0.w; B.c[4] = u1.x; B.c[5] = u1.y; B.c[6] = u1.z; B.c[7] = u1.w;
                res = decide_fast(A, B, P.aabb[r], P.aabb[j], P.area[r] >= 0.f && P.area[j] >= 0.f, P.thr, scratch);
                ++c_clip;
            }
            unsigned hard = __ballot_sync(0xffffffffu, valid && res < 0);
            while (hard) {
                const int src = __ffs(hard) - 1;
                hard &= hard - 1;
                Quad HA, HB;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    HA.c[k] = __shfl_sync(0xffffffffu, A.c[k], src);
                    HB.c[k] = __shfl_sync(0xffffffffu, B.c[k], src);
                }
                // better-ranked box first, as the reference's loops call it: for degenerate pairs the fan sum's rounding
                // residue, and with it the IoU, depends on the order
                const bool s = decide_fp64_warp(HB, HA, P.thr, P.union_mode, lane);
                if (lane == src) { res = s ? 1 : 0; ++c_64; }
            }
            if (!valid) continue;
            if (res) {
                ++c_sup;
                if (atomicExch(&P.status[r], 2) == 0) fs_next[atomicAdd(&P.counts[2 + nxt], 1u)] = r;
            } else if (atomicSub(&P.pending[r], 1) == 1) {
                P.status[r] = 1;
                fk_next[atomicAdd(&P.counts[nxt], 1u)] = r;
            }
        }
        ++round;
        __threadfence();
        grid.sync();
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        c_clip += __shfl_down_sync(0xffffffffu, c_clip, o);
        c_64 += __shfl_down_sync(0xffffffffu, c_64, o);
        c_sup += __shfl_down_sync(0xffffffffu, c_sup, o);
    }
    if (lane == 0 && c_clip) {
        atomicAdd(&P.ctr->pairs_clipped, c_clip);
        atomicAdd(&P.ctr->pairs_fp64, c_64);
        atomicAdd(&P.ctr->suppressing, c_sup);
    }
    if (tid == 0) P.ctr->rounds = round;
}

// no-host-sync callers: make a candidate-list overflow visible on the device (the CSR is consistent but incomplete, so
// boxes that should be suppressed could be kept): status_out = 1
__global__ void nms_export_overflow_kernel(const NmsCounters *ctr, int32_t *status_out)
{
    if (ctr->overflow) *status_out = 1;
}

__global__ void __launch_bounds__(256)
nms_flags_kernel(const uint8_t *__restrict__ status, const int32_t *__restrict__ status_orig, const int32_t *__restrict__ order,
                 const int32_t *__restrict__ rank, int n, int out_order,
                 uint8_t *__restrict__ flags, int64_t *__restrict__ vals)
{
    // status is indexed by rank (COMPAT32); status_orig by original box index (EXACT64)
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    if (out_order == ORP_ORDER_SCORE_DESC) {
        flags[k] = (status_orig ? status_orig[order[k]] : (int32_t)status[k]) == 1;      // k = rank, order[k] = its original index
        vals[k] = order[k];
    } else {
        flags[k] = (status_orig ? status_orig[k] : (int32_t)status[rank[k]]) == 1;
        vals[k] = k;
    }
}

// A cooperative resolve launch of 256-thread blocks: as many as can be co-resident (at most 4 per SM), no more than `need`
static int launch_resolve(const void *kernel, int need, void **args, cudaStream_t st)
{
    int sms = 0, per_sm = 0;
    const int rc = device_sms(sms);
    if (rc) return rc;
    ORP_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0));
    if (per_sm > 4) per_sm = 4;
    int grid = sms * (per_sm > 0 ? per_sm : 1);
    if (grid > need) grid = need;
    ORP_CUDA(cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(256), args, 0, st));
    ORP_LAUNCHED();
    return ORP_OK;
}

// flags_out (optional): uint8 [n], 1 where the box (by ORIGINAL index) survives; when given, keep_out /
// num_out may be NULL and the compaction is skipped (used by the fused head post-processing).
int run_nms(const float *dets, const int32_t *segments, int n, double thr, int iou_mode, int union_mode,
            int order, int64_t *keep_out, int32_t *num_out, cudaStream_t st, uint8_t *flags_out, bool no_sync, int seg_limit,
            int32_t *overflow_out)
{
    if (!segments) seg_limit = 1;
    if (n < 0 || (!flags_out && !num_out) || (n > 0 && (!dets || (!flags_out && !keep_out))))
        return fail(ORP_EINVAL, "orp_rnms: null pointer or negative n");
    if (iou_mode != ORP_NMS_EXACT64 && iou_mode != ORP_NMS_COMPAT32) return fail(ORP_EINVAL, "orp_rnms: bad iou_mode");
    if (union_mode < 0 || union_mode > 3) return fail(ORP_EINVAL, "orp_rnms: bad union_mode");
    int rc = ensure_device();
    if (rc) return rc;
    const bool lazy = (iou_mode == ORP_NMS_EXACT64);
    memset(&g_last_plan, 0, sizeof(g_last_plan));
    g_last_plan.lazy = lazy; g_last_plan.seg_limit = seg_limit; g_last_plan.no_sync = no_sync; g_last_plan.flags_out = flags_out != nullptr;
    g_last_plan.union_mode = union_mode; g_last_plan.order = order; g_last_plan.n = n;
    g_have_plan = true;
    if (n == 0) {
        if (num_out) ORP_CUDA(cudaMemsetAsync(num_out, 0, sizeof(int32_t), st));
        return ORP_OK;
    }
    // conventions that compare every pair: two zero-area boxes may suppress each other wherever they are (orp_b200.h), so
    // they are candidates of each other although the sweep never pairs them
    const bool zero_rule = lazy && (union_mode == ORP_UNION_GUARD || union_mode == ORP_UNION_NAN_SUPPRESSES_ALL);
    // Registration slots per box.  Large single sets (the poly_nms sweep: 10^5 boxes in one segment) are cut into y strips
    // so that a box only meets the boxes of its own strips while walking its x interval; many small segments (a tile:
    // 5 344 boxes per (image, class)) do not need them.  Segment ids must fit 15 bits next to the 16-bit strip index.
    const long long per_seg = seg_limit > 0 ? (long long)n / seg_limit : (long long)n;
    // (an unknown segment bound, seg_limit <= 0, keeps the strip-less layout whose key carries 31 segment bits)
    const int R = (lazy && per_seg >= 16384 && seg_limit > 0 && seg_limit <= 32767) ? 4 : 1;
    const int m = n * R;                                          // registration slots
    // sweep keys: R == 1: (segment : xmin), R == 4: (segment(15) : strip(16) : xmin); only the bits in use are sorted -
    // enough of them that the all-ones keys of padding / non-finite boxes still sort after every real key
    const int sweep_bits = seg_limit > 0 ? (R == 1 ? 32 : 48) + key_bits((uint64_t)seg_limit) : 64;
    // zero-area list sort: as many key bits as the segment ids need, plus the all-ones `none` key of every other box
    const int zbits = seg_limit > 0 ? key_bits((uint64_t)seg_limit) : 32;
    const uint32_t znone = zbits == 32 ? 0xFFFFFFFFu : (uint32_t)((1ull << zbits) - 1);
    // candidate-pair buffer: grows on overflow (one retry costs a host sync; sized to make that rare).  Callers that
    // forbid the host round trip (no_sync) get the overflow reported on the device through overflow_out instead.
    unsigned long long cap = (unsigned long long)n * 256ull;
    if (cap < (1ull << 20)) cap = 1ull << 20;
    const unsigned long long all_pairs = (unsigned long long)n * (unsigned long long)(n - 1) / 2ull;
    if (cap > all_pairs) cap = all_pairs ? all_pairs : 1;
    g_last_plan.R = R; g_last_plan.sweep_bits = sweep_bits;
    g_last_plan.cap_first = g_last_plan.cap_final = (int64_t)cap;
    Scratch S(st);
    const int T = 256, G = ceil_div(n, T), GM = ceil_div(m, T);
    // both modes.  iota: the rank sort's values, then (EXACT64) the registrations' box ids; v01 / v23: vertices by original
    // index (EXACT64) or by rank (COMPAT32); list_len: per box, the edges that name it first = the length of its CSR list
    uint32_t *score_key = S.get<uint32_t>(n), *score_key2 = S.get<uint32_t>(n);
    int32_t *iota = S.get<int32_t>(m), *order_r = S.get<int32_t>(n), *rank = S.get<int32_t>(n);
    float4 *v01 = S.get<float4>(n), *v23 = S.get<float4>(n);
    int32_t *list_len = S.get<int32_t>(n + 1), *offs = S.get<int32_t>(n + 1), *cursor = S.get<int32_t>(n + 1);
    uint8_t *flags = flags_out ? flags_out : S.get<uint8_t>(n);
    int64_t *vals = S.get<int64_t>(n);
    NmsCounters *ctr = S.get<NmsCounters>(1);
    // EXACT64: per box AABB and area, the registrations in sweep order, the lazy resolve's state
    uint64_t *sweep_key = lazy ? S.get<uint64_t>(m) : nullptr, *sweep_key2 = lazy ? S.get<uint64_t>(m) : nullptr;
    int32_t *perm = lazy ? S.get<int32_t>(m) : nullptr, *nvalid = lazy ? S.get<int32_t>(1) : nullptr;
    float4 *baabb = lazy ? S.get<float4>(n) : nullptr, *aabb_s = lazy ? S.get<float4>(m) : nullptr;
    int4 *meta_s = lazy ? S.get<int4>(m) : nullptr;
    float *area = lazy ? S.get<float>(n) : nullptr;
    NmsGlobal *glob = lazy ? S.get<NmsGlobal>(1) : nullptr;
    unsigned int *qcount = lazy ? S.get<unsigned int>(6) : nullptr;          // frontier / queue fills of the lazy resolve
    int32_t *worklist = lazy ? S.get<int32_t>(4 * (size_t)n) : nullptr;   // kept and suppressed frontiers, [2][n] each
    int32_t *status32 = lazy ? S.get<int32_t>(n) : nullptr, *pending = lazy ? S.get<int32_t>(n) : nullptr;
    int32_t *zlist = zero_rule ? S.get<int32_t>(n) : nullptr, *zpos = zero_rule ? S.get<int32_t>(n) : nullptr;
    int32_t *zhi = zero_rule ? S.get<int32_t>(n) : nullptr, *zbetter = zero_rule ? S.get<int32_t>(n) : nullptr;
    // COMPAT32: segment ids in rank order, the rescanning resolve's status (by rank) and change flags
    int32_t *sg = lazy ? nullptr : S.get<int32_t>(n);
    uint8_t *status = lazy ? nullptr : S.get<uint8_t>(n);
    int *changed = lazy ? nullptr : S.get<int>(2);
    if (!ctr || !vals || !flags || (lazy && (!worklist || !status32 || !pending || !meta_s || !qcount || !glob)) ||
        (zero_rule && (!zlist || !zpos || !zhi || !zbetter)) || (!lazy && (!sg || !status || !changed)))
        return fail(ORP_ECUDA, "orp_rnms: scratch allocation failed");

    size_t tb1 = 0, tb2 = 0, tb3 = 0, tb4 = 0, tb5 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb1, score_key, score_key2, iota, order_r, n, 0, 32, st);
    if (lazy) cub::DeviceRadixSort::SortPairs(nullptr, tb2, sweep_key, sweep_key2, iota, perm, m, 0, sweep_bits, st);
    if (zero_rule) cub::DeviceRadixSort::SortPairs(nullptr, tb5, score_key, score_key2, order_r, zlist, n, 0, zbits, st);
    cub::DeviceScan::ExclusiveSum(nullptr, tb3, list_len, offs, n + 1, st);
    if (keep_out && num_out) cub::DeviceSelect::Flagged(nullptr, tb4, vals, flags, keep_out, num_out, n, st);
    size_t tb = tb1 > tb2 ? tb1 : tb2;
    tb = tb > tb3 ? tb : tb3;
    tb = tb > tb4 ? tb : tb4;
    tb = tb > tb5 ? tb : tb5;
    uint8_t *tmp = S.get<uint8_t>(tb);
    if (!tmp) return fail(ORP_ECUDA, "orp_rnms: scratch allocation failed");

    ORP_CUDA(cudaMemsetAsync(ctr, 0, sizeof(NmsCounters), st));
    ORP_CUDA(cudaMemsetAsync(list_len, 0, sizeof(int32_t) * (size_t)(n + 1), st));
    ORP_CUDA(cudaMemsetAsync(cursor, 0, sizeof(int32_t) * (size_t)(n + 1), st));

    nms_prep_kernel<<<G, T, 0, st>>>(dets, n, score_key, iota);
    ORP_LAUNCHED();
    ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb1, score_key, score_key2, iota, order_r, n, 0, 32, st));
    count_launches(4);
    nms_rank_kernel<<<G, T, 0, st>>>(order_r, n, rank);
    ORP_LAUNCHED();

    if (lazy) {
        ORP_CUDA(cudaMemsetAsync(pending, 0, sizeof(int32_t) * (size_t)n, st));
        ORP_CUDA(cudaMemsetAsync(glob, 0, sizeof(NmsGlobal), st));
        ORP_CUDA(cudaMemsetAsync(&glob->ymin_key, 0xFF, sizeof(glob->ymin_key), st));   // the identity of atomicMin
        nms_boxes_kernel<<<G, T, 0, st>>>(dets, n, baabb, v01, v23, area, glob);
        ORP_LAUNCHED();
        nms_regs_kernel<<<G, T, 0, st>>>(baabb, segments, n, R, glob, sweep_key, iota);
        ORP_LAUNCHED();
        ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb2, sweep_key, sweep_key2, iota, perm, m, 0, sweep_bits, st));
        count_launches((sweep_bits + 7) / 8);
        nms_slots_kernel<<<GM, T, 0, st>>>(sweep_key2, perm, baabb, area, rank, m, aabb_s, meta_s, nvalid);
        ORP_LAUNCHED();
        if (zero_rule) {
            ORP_CUDA(cudaMemsetAsync(zpos, 0xFF, sizeof(int32_t) * (size_t)n, st));   // -1: not a zero-area box
            // score keys are free after the rank sort: they carry the zero-area list keys
            nms_zero_keys_kernel<<<G, T, 0, st>>>(order_r, segments, v01, v23, glob, n, znone, area, score_key);
            ORP_LAUNCHED();
            ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb5, score_key, score_key2, order_r, zlist, n, 0, zbits, st));
            count_launches((zbits + 7) / 8);
            nms_zero_list_kernel<<<G, T, 0, st>>>(score_key2, zlist, n, znone, zpos, zhi, zbetter);
            ORP_LAUNCHED();
        }
    } else {
        nms_gather_kernel<<<G, T, 0, st>>>(dets, segments, order_r, n, v01, v23, sg);
        ORP_LAUNCHED();
    }

    int2 *edges = nullptr;
    for (int attempt = 0; attempt < 6; ++attempt) {
        g_last_plan.attempts = attempt + 1;
        g_last_plan.cap_final = (int64_t)cap;
        // the buffer turns into the resolve's work queue; the zero-area lists can add one pair per box and round to it
        edges = S.get<int2>(cap + (zero_rule ? (unsigned long long)n : 0ull));
        if (!edges) return fail(ORP_ECUDA, "orp_rnms: edge buffer allocation failed");
        if (lazy) {
            SweepParams P{aabb_s, meta_s, v01, v23, nvalid, glob, R, edges, list_len, pending, cap, ctr, thr, union_mode};
            int grid = ceil_div(m, kSweepWarps);
            const int maxgrid = kNumSMs * 8 * 4;
            if (grid > maxgrid) grid = maxgrid;
            if (g_timing) {
                if (!g_ev[0]) { ORP_CUDA(cudaEventCreate(&g_ev[0])); ORP_CUDA(cudaEventCreate(&g_ev[1])); }
                ORP_CUDA(cudaEventRecord(g_ev[0], st));
            }
            nms_sweep_kernel<<<grid, kSweepWarps * 32, 0, st>>>(P);
            ORP_LAUNCHED();
            if (g_timing) ORP_CUDA(cudaEventRecord(g_ev[1], st));
        } else {
            const long long nb = (n + 63) / 64;
            const long long tiles = nb * (nb + 1) / 2;
            if (tiles > 2147483647LL) return fail(ORP_EINVAL, "orp_rnms: n too large for COMPAT32 mode");
            nms_compat_tiles_kernel<<<(unsigned)tiles, 64, 0, st>>>(v01, v23, sg, n, (float)thr, union_mode, edges,
                                                                    list_len, cap, ctr);
            ORP_LAUNCHED();
        }
        if (cap >= all_pairs || no_sync) break;   // cannot overflow / caller forbids the host round trip
        // overflow check needs the host; it is the only sync of the call and only happens when
        // the edge list could in principle exceed its capacity
        NmsCounters h;
        ORP_CUDA(cudaMemcpyAsync(&h, ctr, sizeof(h), cudaMemcpyDeviceToHost, st));
        ORP_CUDA(cudaStreamSynchronize(st));
        if (!h.overflow) break;
        if (attempt == 5) return fail(ORP_EOVERFLOW, "orp_rnms: edge buffer overflow");
        cap = h.edges + h.edges / 8 + 1024;
        if (cap > all_pairs) cap = all_pairs;
        ORP_CUDA(cudaMemsetAsync(ctr, 0, sizeof(NmsCounters), st));
        ORP_CUDA(cudaMemsetAsync(list_len, 0, sizeof(int32_t) * (size_t)(n + 1), st));
        if (lazy) ORP_CUDA(cudaMemsetAsync(pending, 0, sizeof(int32_t) * (size_t)n, st));
    }
    if (zero_rule) {
        nms_zero_pending_kernel<<<G, T, 0, st>>>(zpos, zbetter, n, pending);
        ORP_LAUNCHED();
    }

    ORP_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb3, list_len, offs, n + 1, st));
    count_launches(2);
    int32_t *adj = S.get<int32_t>(cap);
    if (!adj) return fail(ORP_ECUDA, "orp_rnms: adjacency allocation failed");
    nms_scatter_kernel<<<kNumSMs * 8, 256, 0, st>>>(edges, ctr, cap, offs, cursor, adj);
    ORP_LAUNCHED();
    if (lazy) {
        ORP_CUDA(cudaMemsetAsync(status32, 0, sizeof(int32_t) * (size_t)n, st));
        ORP_CUDA(cudaMemsetAsync(qcount, 0, 6 * sizeof(unsigned int), st));
        // the candidate buffer is free once scattered into the CSR: it becomes the work queue; after the scatter
        // `cursor` holds every list's length
        LazyParams LP{offs, adj, cursor, n, status32, pending, ctr, qcount, worklist, worklist + 2 * (size_t)n, edges,
                      baabb, v01, v23, area, thr, union_mode, zlist, zpos, zhi};
        void *args[] = {&LP};
        rc = launch_resolve((const void *)nms_resolve_lazy_kernel, ceil_div(n, 8), args, st);   // a warp per frontier box
    } else {
        ORP_CUDA(cudaMemsetAsync(status, 0, (size_t)n, st));
        ORP_CUDA(cudaMemsetAsync(changed, 0, 2 * sizeof(int), st));
        // a pointer and its cv-qualified version share one representation: these are the kernel's parameters
        void *args[] = {&offs, &adj, &n, &status, &changed, &ctr};
        rc = launch_resolve((const void *)nms_resolve_kernel, ceil_div(n, 256), args, st);
    }
    if (rc) return rc;
    if (overflow_out) {
        nms_export_overflow_kernel<<<1, 1, 0, st>>>(ctr, overflow_out);
        ORP_LAUNCHED();
    }
    // EXACT64: status32 is indexed by original box index; COMPAT32: status by rank
    nms_flags_kernel<<<G, T, 0, st>>>(status, status32, order_r, rank, n, flags_out ? ORP_ORDER_INDEX_ASC : order, flags, vals);
    ORP_LAUNCHED();
    if (keep_out && num_out) {
        if (flags_out && order != ORP_ORDER_INDEX_ASC) return fail(ORP_EINVAL, "orp_rnms: flags_out needs index order");
        ORP_CUDA(cub::DeviceSelect::Flagged(tmp, tb4, vals, flags, keep_out, num_out, n, st));
        count_launches(3);
    }

    // stash the counters for orp_rnms_last_stats (async copy into pinned memory)
    if (!g_stats_pinned) ORP_CUDA(cudaHostAlloc(&g_stats_pinned, sizeof(NmsCounters), cudaHostAllocDefault));
    ORP_CUDA(cudaMemcpyAsync(g_stats_pinned, ctr, sizeof(NmsCounters), cudaMemcpyDeviceToHost, st));
    g_last_n = n;
    return ORP_OK;
}

}  // namespace orp

extern "C" int orp_rnms(const float *dets, const int32_t *segments, int n, double iou_thr, int iou_mode,
                        int union_mode, int order, int64_t *keep_out, int32_t *num_out, void *stream)
{
    return orp::run_nms(dets, segments, n, iou_thr, iou_mode, union_mode, order, keep_out, num_out,
                        static_cast<cudaStream_t>(stream), nullptr, false, 0, nullptr);
}

extern "C" int orp_rnms_last_sweep_ms(float *ms)
{
    if (!ms) return orp::fail(ORP_EINVAL, "orp_rnms_last_sweep_ms: null");
    if (!orp::g_timing || !orp::g_ev[0]) return orp::fail(ORP_EINVAL, "orp_rnms_last_sweep_ms: timing is off");
    ORP_CUDA(cudaEventSynchronize(orp::g_ev[1]));
    ORP_CUDA(cudaEventElapsedTime(ms, orp::g_ev[0], orp::g_ev[1]));
    return ORP_OK;
}

extern "C" int orp_rnms_last_stats(orp_nms_stats *out)
{
    if (!out) return orp::fail(ORP_EINVAL, "orp_rnms_last_stats: null");
    if (!orp::g_stats_pinned) return orp::fail(ORP_EINVAL, "orp_rnms_last_stats: no previous call");
    const orp::NmsCounters &c = *orp::g_stats_pinned;
    out->pairs_total = (int64_t)c.pairs_swept;
    out->pairs_aabb = (int64_t)c.pairs_aabb;
    out->pairs_clipped = (int64_t)c.pairs_clipped;
    out->pairs_fp64 = (int64_t)c.pairs_fp64;
    out->edges = (int64_t)c.edges;
    out->suppressing = (int64_t)c.suppressing;
    out->overflow = c.overflow;
    out->rounds = c.rounds;
    out->n = orp::g_last_n;
    return ORP_OK;
}

extern "C" int orp_rnms_last_plan(orp_rnms_plan *out)
{
    if (!out) return orp::fail(ORP_EINVAL, "orp_rnms_last_plan: null");
    if (!orp::g_have_plan) return orp::fail(ORP_EINVAL, "orp_rnms_last_plan: no previous call");
    *out = orp::g_last_plan;
    return ORP_OK;
}

extern "C" int orp_poly_nms_host(int *keep_out, int *num_out, const float *polys_host, int polys_num,
                                 int polys_dim, float nms_overlap_thresh, int device_id)
{
    using namespace orp;
    if (polys_dim != 9) return fail(ORP_EINVAL, "orp_poly_nms_host: polys_dim must be 9");
    if (polys_num < 0 || !num_out || (polys_num > 0 && (!keep_out || !polys_host)))
        return fail(ORP_EINVAL, "orp_poly_nms_host: bad arguments");
    if (polys_num == 0) { *num_out = 0; return ORP_OK; }
    int prev = 0;
    ORP_CUDA(cudaGetDevice(&prev));
    ORP_CUDA(cudaSetDevice(device_id));
    cudaStream_t st;
    ORP_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    const int rc = [&]() -> int {
        Scratch S(st);
        float *d = S.get<float>(9 * (size_t)polys_num);
        int64_t *k = S.get<int64_t>(polys_num);
        int32_t *cnt = S.get<int32_t>(1);
        if (!d || !k || !cnt) return fail(ORP_ECUDA, "orp_poly_nms_host: alloc");
        ORP_CUDA(cudaMemcpyAsync(d, polys_host, sizeof(float) * 9 * (size_t)polys_num, cudaMemcpyHostToDevice, st));
        // the caller sorted by score already (poly_nms.pyx:19-21); our stable descending sort
        // reproduces that order exactly, so SCORE_DESC output == positions in the sorted input
        const int err = run_nms(d, nullptr, polys_num, (double)nms_overlap_thresh, ORP_NMS_EXACT64, ORP_UNION_GUARD,
                                ORP_ORDER_SCORE_DESC, k, cnt, st, nullptr, false, 1, nullptr);
        if (err) return err;
        int32_t hc = 0;
        ORP_CUDA(cudaMemcpyAsync(&hc, cnt, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        ORP_CUDA(cudaStreamSynchronize(st));
        std::vector<int64_t> hk(hc > 0 ? hc : 1);
        ORP_CUDA(cudaMemcpyAsync(hk.data(), k, sizeof(int64_t) * (size_t)hc, cudaMemcpyDeviceToHost, st));
        ORP_CUDA(cudaStreamSynchronize(st));
        for (int i = 0; i < hc; ++i) keep_out[i] = (int)hk[i];
        *num_out = hc;
        return ORP_OK;
    }();
    cudaStreamSynchronize(st);
    cudaStreamDestroy(st);
    cudaSetDevice(prev);
    return rc;
}
