// evaluation.cu - DOTA Task1 evaluation on the device (orp_dota_eval_task1).
//
// Replaces the per-class Python loop of voc_eval (DOTA_devkit/dota_evaluation_task1.py:87-248) for every class at once.
// The loop's one sequential dependency is the `det` flag a detection sets on its target; the target itself (jmax, the
// argmax of IoU over the ground truth of the detection's image and class) does not depend on earlier claims, because
// VOC matching never falls back to the next-best box.  So the evaluation is:
//
//   order  stable radix sorts: score descending, then class ascending -> position p (the rank inside a class)
//   match  detections bucketed by (class, image); a CTA stages the bucket's ground truth in shared memory (looping over
//          stages) and computes ovmax / jmax per detection: the "+1 pixel" AABB prefilter of :176-205 operation for
//          operation, then iou_poly(gt, det) (ref_quad_pair<double>, :211) with numpy's max / argmax semantics
//   claim  atomicMin(claim[jmax], p) for every hit on a non-difficult box; the smallest position is the true positive
//   pr     one scan of the packed (tp, fp) counts, rec / prec with the IEEE operations of :239-245
//   ap     voc_ap (:53-84) per class, one CTA each
//
// The cost is the fp64 clipping of the prefilter's surviving pairs plus four radix sorts over the inputs.
#include <cub/cub.cuh>
#include <float.h>

#include "common.cuh"
#include "geom.cuh"

namespace orp {
namespace {

constexpr int kEvalThreads = 256;   // detections per CTA of the match kernel, threads of every kernel here
constexpr int kGtStage = 128;       // ground-truth boxes per shared-memory stage of the match kernel

enum : uint8_t { kFalsePos = 0, kDifficultHit = 1, kCandidate = 2 };

struct Thresholds { double t[11]; };

// numpy's np.maximum / np.minimum / np.min: a NaN operand wins
__device__ __forceinline__ double np_max(double a, double b) { return (a != a) ? a : ((b != b) ? b : (a >= b ? a : b)); }
__device__ __forceinline__ double np_min(double a, double b) { return (a != a) ? a : ((b != b) ? b : (a <= b ? a : b)); }

// (xmin, ymin, xmax, ymax) of a quadrilateral as np.min / np.max over its x and y coordinates (:179-186)
__device__ __forceinline__ double4 quad_aabb(const double *q)
{
    double4 b;
    b.x = np_min(np_min(q[0], q[2]), np_min(q[4], q[6]));
    b.y = np_min(np_min(q[1], q[3]), np_min(q[5], q[7]));
    b.z = np_max(np_max(q[0], q[2]), np_max(q[4], q[6]));
    b.w = np_max(np_max(q[1], q[3]), np_max(q[5], q[7]));
    return b;
}

// BBGT_keep_mask of :188-203 for one (gt, det) pair: `inters / uni > 0`, every operation rounded on its own
__device__ __forceinline__ bool aabb_keep(double4 g, double4 b)
{
    const double ixmin = np_max(g.x, b.x), iymin = np_max(g.y, b.y);
    const double ixmax = np_min(g.z, b.z), iymax = np_min(g.w, b.w);
    const double iw = np_max(__dadd_rn(__dsub_rn(ixmax, ixmin), 1.0), 0.0);
    const double ih = np_max(__dadd_rn(__dsub_rn(iymax, iymin), 1.0), 0.0);
    const double inters = __dmul_rn(iw, ih);
    const double ab = __dmul_rn(__dadd_rn(__dsub_rn(b.z, b.x), 1.0), __dadd_rn(__dsub_rn(b.w, b.y), 1.0));
    const double ag = __dmul_rn(__dadd_rn(__dsub_rn(g.z, g.x), 1.0), __dadd_rn(__dsub_rn(g.w, g.y), 1.0));
    const double uni = __dsub_rn(__dadd_rn(ab, ag), inters);
    return __ddiv_rn(inters, uni) > 0.0;
}

// score -> ascending key of the DESCENDING score order; NaN last (np.argsort(-confidence)), -0.0 == +0.0
__device__ __forceinline__ uint64_t score_desc_key(double s)
{
    if (s != s) return ~0ull;
    if (s == 0.0) s = 0.0;
    uint64_t u = (uint64_t)__double_as_longlong(s);
    u = (u >> 63) ? ~u : (u | (1ull << 63));
    return ~u;
}

__device__ __forceinline__ int lower_bound_u32(const uint32_t *a, int n, uint32_t v)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kEvalThreads)
eval_det_prep_kernel(const double *__restrict__ score, int nd, uint64_t *__restrict__ key, int32_t *__restrict__ iota)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nd; i += gridDim.x * blockDim.x) {
        key[i] = score_desc_key(score[i]);
        iota[i] = i;
    }
}

// class key of each detection in score order; ids outside [0, ncls) get ncls and sort after every class
__global__ void __launch_bounds__(kEvalThreads)
eval_class_key_kernel(const int32_t *__restrict__ det_cls, const int32_t *__restrict__ by_score, int nd, int ncls,
                      uint32_t *__restrict__ ckey)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nd; i += gridDim.x * blockDim.x) {
        const int c = det_cls[by_score[i]];
        ckey[i] = (c >= 0 && c < ncls) ? (uint32_t)c : (uint32_t)ncls;
    }
}

__global__ void __launch_bounds__(kEvalThreads)
eval_class_offsets_kernel(const uint32_t *__restrict__ ckey, int nd, int ncls, int64_t *__restrict__ cls_off)
{
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= ncls; c += gridDim.x * blockDim.x)
        cls_off[c] = lower_bound_u32(ckey, nd, (uint32_t)c);
}

// (class, image) bucket of the detection at class-score position p; buckets of out-of-range ids are `none` (= nseg)
__global__ void __launch_bounds__(kEvalThreads)
eval_det_seg_kernel(const int32_t *__restrict__ det_img, const int32_t *__restrict__ order, const uint32_t *__restrict__ ckey,
                    int nd, int ncls, int nimg, uint32_t *__restrict__ seg, int32_t *__restrict__ iota)
{
    const uint32_t none = (uint32_t)ncls * (uint32_t)nimg;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < nd; p += gridDim.x * blockDim.x) {
        const uint32_t c = ckey[p];
        const int im = det_img[order[p]];
        seg[p] = (c < (uint32_t)ncls && im >= 0 && im < nimg) ? c * (uint32_t)nimg + (uint32_t)im : none;
        iota[p] = p;
    }
}

__global__ void __launch_bounds__(kEvalThreads)
eval_gt_seg_kernel(const int32_t *__restrict__ gt_cls, const int32_t *__restrict__ gt_img, int ng, int ncls, int nimg,
                   uint32_t *__restrict__ seg, int32_t *__restrict__ iota)
{
    const uint32_t none = (uint32_t)ncls * (uint32_t)nimg;
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < ng; g += gridDim.x * blockDim.x) {
        const int c = gt_cls[g], im = gt_img[g];
        seg[g] = (c >= 0 && c < ncls && im >= 0 && im < nimg) ? (uint32_t)c * (uint32_t)nimg + (uint32_t)im : none;
        iota[g] = g;
    }
}

// ground truth in bucket order (input order inside a bucket: the stable sort keeps it, and np.argmax's first maximum
// refers to it); for the VOC matching (kVoc) also npos per class (:139) and the claims reset
template <bool kVoc>
__global__ void __launch_bounds__(kEvalThreads)
eval_gt_gather_kernel(const double *__restrict__ gt_quad, const uint8_t *__restrict__ gt_difficult,
                      const int32_t *__restrict__ gt_cls, const int32_t *__restrict__ gorder, const uint32_t *__restrict__ gseg,
                      int ng, int ncls, int nimg, double *__restrict__ gq, double4 *__restrict__ gbox,
                      uint8_t *__restrict__ gdiff, unsigned long long *__restrict__ npos, int32_t *__restrict__ claim)
{
    const uint32_t none = (uint32_t)ncls * (uint32_t)nimg;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < ng; k += gridDim.x * blockDim.x) {
        const int g = gorder[k];
        double q[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { q[i] = gt_quad[(size_t)g * 8 + i]; gq[(size_t)k * 8 + i] = q[i]; }
        gbox[k] = quad_aabb(q);
        if constexpr (kVoc) {
            const uint8_t d = gt_difficult[g] != 0;
            gdiff[k] = d;
            claim[k] = INT_MAX;
            if (gseg[k] != none && !d) atomicAdd(&npos[gt_cls[g]], 1ull);
        }
    }
}

// ovmax / jmax of every detection (:166-220).  kVoc: the claims of :222-228 and a status per position; otherwise (the
// mAOE matching, mAOE_evaluation.py:114-160: no difficult flags, no claims) jm[p] = jmax when ovmax > ovthresh, else -1.
// CTA = kEvalThreads consecutive detections of the bucket order; it walks the buckets they cover, staging each bucket's
// ground truth kGtStage boxes at a time.  One CTA per SM: the call to the fp64 clipping (ref_quad_pair) needs ~190
// registers to run without spills.
template <bool kVoc>
__global__ void __launch_bounds__(kEvalThreads, 1)
eval_match_kernel(const uint32_t *__restrict__ dseg, const int32_t *__restrict__ dpos, const int32_t *__restrict__ order,
                  const double *__restrict__ det_quad, int nd, const uint32_t *__restrict__ gseg, const double *__restrict__ gq,
                  const double4 *__restrict__ gbox, const uint8_t *__restrict__ gdiff, int ng, uint32_t none, double ovthresh,
                  int32_t *__restrict__ claim, int32_t *__restrict__ jm, uint8_t *__restrict__ status)
{
    __shared__ double s_det[kEvalThreads][8];
    __shared__ double s_gq[kGtStage][8];
    __shared__ double4 s_gbox[kGtStage];
    __shared__ uint32_t s_key[kEvalThreads];
    __shared__ int s_lo, s_hi;
    __shared__ uint32_t s_next;

    const int t = threadIdx.x;
    const int i = blockIdx.x * kEvalThreads + t;
    const bool live = i < nd;
    const uint32_t key = live ? dseg[i] : none;
    const int p = live ? dpos[i] : 0;
    double4 bb = make_double4(0, 0, 0, 0);
    if (live) {
        const int d = order[p];
#pragma unroll
        for (int k = 0; k < 8; ++k) s_det[t][k] = det_quad[(size_t)d * 8 + k];
        bb = quad_aabb(s_det[t]);
    }
    s_key[t] = key;
    double ov = -INFINITY;   // ovmax = -np.inf (:169)
    int jmax = -1;           // global index of the target in bucket order
    bool nan_seen = false;
    __syncthreads();

    uint32_t cur = s_key[0];
    while (cur != none) {
        if (t == 0) {
            s_lo = lower_bound_u32(gseg, ng, cur);
            s_hi = lower_bound_u32(gseg, ng, cur + 1);
        }
        __syncthreads();
        const int lo = s_lo, hi = s_hi;
        for (int base = lo; base < hi; base += kGtStage) {
            const int cnt = min(kGtStage, hi - base);
            for (int e = t; e < cnt * 8; e += kEvalThreads) s_gq[e >> 3][e & 7] = gq[(size_t)base * 8 + e];
            for (int e = t; e < cnt; e += kEvalThreads) s_gbox[e] = gbox[base + e];
            __syncthreads();
            if (key == cur) {
                for (int k = 0; k < cnt; ++k) {
                    if (!aabb_keep(s_gbox[k], bb)) continue;
                    if (nan_seen) continue;            // np.max / np.argmax: the first NaN is final
                    const PairRes<double> r = ref_quad_pair<double>(s_gq[k], s_det[t]);
                    const double v = iou_from<double>(r, ORP_UNION_NAN_KEEPS);
                    if (v != v) { nan_seen = true; ov = v; jmax = base + k; }
                    else if (jmax < 0 || v > ov) { ov = v; jmax = base + k; }
                }
            }
            __syncthreads();
        }
        // next bucket: the key that starts the next run of this CTA's sorted keys
        if (t == 0) s_next = none;
        __syncthreads();
        if (t > 0 && key > cur && s_key[t - 1] <= cur) s_next = key;
        __syncthreads();
        cur = s_next;
        __syncthreads();
    }

    if (!live) return;
    if constexpr (kVoc) {
        uint8_t st = kFalsePos;
        if (jmax >= 0 && ov > ovthresh) {
            if (gdiff[jmax]) st = kDifficultHit;
            else { st = kCandidate; atomicMin(&claim[jmax], p); }
        }
        jm[p] = jmax;
        status[p] = st;
    } else {
        jm[p] = (jmax >= 0 && ov > ovthresh) ? jmax : -1;
    }
}

// tp / fp of every position, packed as (tp << 32) | fp for one scan
__global__ void __launch_bounds__(kEvalThreads)
eval_tpfp_kernel(const uint8_t *__restrict__ status, const int32_t *__restrict__ jm, const int32_t *__restrict__ claim, int nd,
                 unsigned long long *__restrict__ tpfp)
{
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < nd; p += gridDim.x * blockDim.x) {
        const uint8_t st = status[p];
        unsigned long long v = 0;
        if (st == kFalsePos) v = 1;
        else if (st == kCandidate) v = claim[jm[p]] == p ? (1ull << 32) : 1ull;
        tpfp[p] = v;
    }
}

// rec = tp / float(npos), prec = tp / np.maximum(tp + fp, eps) (:239-245) from the running counts of the position's class
__global__ void __launch_bounds__(kEvalThreads)
eval_pr_kernel(const unsigned long long *__restrict__ cum, const uint32_t *__restrict__ ckey,
               const int64_t *__restrict__ cls_off, const unsigned long long *__restrict__ npos, int nd, int ncls,
               double *__restrict__ rec, double *__restrict__ prec)
{
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < nd; p += gridDim.x * blockDim.x) {
        const uint32_t c = ckey[p];
        if (c >= (uint32_t)ncls) { rec[p] = prec[p] = __longlong_as_double(0x7ff8000000000000ll); continue; }
        const int64_t start = cls_off[c];
        const unsigned long long v = cum[p] - (start > 0 ? cum[start - 1] : 0ull);
        const double tp = (double)(v >> 32), fp = (double)(v & 0xffffffffull);
        rec[p] = __ddiv_rn(tp, (double)npos[c]);
        const double den = __dadd_rn(tp, fp);
        prec[p] = __ddiv_rn(tp, den >= DBL_EPSILON ? den : DBL_EPSILON);
    }
}

// voc_ap (:53-84) per class, one CTA each
__global__ void __launch_bounds__(kEvalThreads)
eval_ap_kernel(const double *__restrict__ rec, const double *__restrict__ prec, const int64_t *__restrict__ cls_off,
               int use_07_metric, Thresholds thr, double *__restrict__ ap)
{
    using Reduce = cub::BlockReduce<double, kEvalThreads>;
    using Scan = cub::BlockScan<double, kEvalThreads>;
    __shared__ union { typename Reduce::TempStorage r; typename Scan::TempStorage s; } tmp;
    __shared__ double s_carry;
    const int c = blockIdx.x, t = threadIdx.x;
    const int64_t a = cls_off[c], n = cls_off[c + 1] - a;
    const double *r = rec + a, *pr = prec + a;
    auto dmax = [](double x, double y) { return x >= y ? x : y; };   // prec is never NaN

    if (use_07_metric) {
        // for t in np.arange(0., 1.1, 0.1): p = max(prec[rec >= t]) or 0; ap = ap + p / 11.
        double acc = 0.0;
        for (int k = 0; k < 11; ++k) {
            double m = -INFINITY;
            for (int64_t q = t; q < n; q += kEvalThreads)
                if (r[q] >= thr.t[k]) m = dmax(m, pr[q]);
            m = Reduce(tmp.r).Reduce(m, dmax);
            if (t == 0) acc = __dadd_rn(acc, __ddiv_rn(m == -INFINITY ? 0.0 : m, 11.0));
            __syncthreads();
        }
        if (t == 0) ap[c] = acc;
        return;
    }
    // area: mrec = [0, rec, 1], mpre = [0, prec, 0] with its suffix-max envelope; sum of (mrec[i+1] - mrec[i]) * mpre[i+1]
    // over the points where mrec changes.  Chunks from the end; thread j holds element b-1-j, so an inclusive max scan
    // over the threads is the suffix max inside the chunk.
    double part = 0.0;
    if (t == 0) s_carry = 0.0;   // mpre's trailing sentinel
    __syncthreads();
    for (int64_t b = n; b > 0; b -= kEvalThreads) {
        const int64_t q = b - 1 - t;
        const bool in = q >= 0;
        double env = in ? pr[q] : 0.0;
        Scan(tmp.s).InclusiveScan(env, env, dmax);
        const double carry = s_carry;
        env = dmax(env, carry);
        if (in) {
            const double cur = r[q], prev = q > 0 ? r[q - 1] : 0.0;
            if (cur != prev) part = __dadd_rn(part, __dmul_rn(__dsub_rn(cur, prev), env));
        }
        __syncthreads();
        if (t == (b < kEvalThreads ? b : kEvalThreads) - 1) s_carry = env;   // the chunk's first element
        __syncthreads();
    }
    double sum = Reduce(tmp.r).Sum(part);
    if (t == 0) {
        const double last = n > 0 ? r[n - 1] : 0.0;   // the final point (1, 0)
        if (last != 1.0) sum = __dadd_rn(sum, __dmul_rn(__dsub_rn(1.0, last), 0.0));
        ap[c] = sum;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// poly2rbox_single_v3 (DOTA_devkit/dota_poly2rbox.py:128-190) and the mAOE (mAOE_evaluation.py)
// ---------------------------------------------------------------------------------------------------------------------

constexpr double kQuarterPi = 0.78539816339744830962;   // np.pi / 4; k * kQuarterPi is exact for k = 1 .. 5

struct RBox { double x, y, w, h, a; };

// np.arctan2 of a float32 direction widened to double.  Directions on an axis or a diagonal return numpy's constants
// k * pi / 4: norm_angle wraps at -pi/4 and 3pi/4, so these must be bit-exact (3pi/4 becomes -pi/4).  Any other float32
// direction is at least ~2^-25 rad from those, where CUDA's atan2 (<= 2 ulp) cannot move it across the wrap.
__device__ __forceinline__ double np_atan2(double y, double x)
{
    if (x != x || y != y) return x + y;
    if (y == 0.0) return (x > 0.0 || (x == 0.0 && !signbit(x))) ? copysign(0.0, y) : copysign(4.0 * kQuarterPi, y);
    if (x == 0.0) return copysign(2.0 * kQuarterPi, y);
    if (fabs(x) == fabs(y)) return copysign(x > 0.0 ? kQuarterPi : 3.0 * kQuarterPi, y);
    return atan2(y, x);
}

// norm_angle(a) = (a + pi/4) % pi - pi/4 with numpy's floor mod (npy_divmod): range [-pi/4, 3pi/4)
__device__ __forceinline__ double norm_angle(double a)
{
    const double pi = 4.0 * kQuarterPi;
    double m = fmod(__dsub_rn(a, -kQuarterPi), pi);   // fmod is exact
    if (m != 0.0) { if (m < 0.0) m = __dadd_rn(m, pi); }
    else m = 0.0;
    return __dadd_rn(m, -kQuarterPi);
}

// the exact |norm_angle| of direction (x, y) as a vector of angle in [0, 3pi/4): turned into norm_angle's half-plane,
// then mirrored into y >= 0
__device__ __forceinline__ void fold_direction(float x, float y, float &u, float &v)
{
    if (!(x > -y || (x == -y && x > 0.f))) { x = -x; y = -y; }
    u = x;
    v = fabsf(y);
}

// abs(a1) > abs(a2) for a1 = norm_angle(atan2(y1, x1)), a2 = norm_angle(atan2(y2, x2)).  Outside a band of ~45 ulp the
// doubles decide: there numpy's and CUDA's atan2 (each within a few ulp of the exact angle) agree on the order.  Inside
// it the order of the exact angles decides - the sign of a cross product of float32 values, whose fp64 products are exact
// - so exact ties (squares, mirrored edges) go to edge 1->2 as the reference's `>` sends them.
__device__ __forceinline__ bool abs_angle_greater(double a1, double a2, float x1, float y1, float x2, float y2)
{
    const double d = __dsub_rn(fabs(a1), fabs(a2));
    if (!(fabs(d) <= 1e-14)) return d > 0.0;   // also NaN: the reference's comparison is false
    float u1, v1, u2, v2;
    fold_direction(x1, y1, u1, v1);
    fold_direction(x2, y2, u2, v2);
    if (x2 == 0.f && y2 == 0.f) return v1 > 0.f;   // angle 0
    return __dmul_rn((double)u2, (double)v1) > __dmul_rn((double)v2, (double)u1);
}

// poly2rbox_single_v3: the quad cast to float32, edges and ratio in float32 (no FMA), angles of the float32 differences
// widened to double, builtin max / min (a NaN edge is kept when it comes first), `ratio < 1.15` in float32
__device__ RBox poly2rbox_v3(const double *q)
{
    float p[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) p[i] = __double2float_rn(q[i]);
    const float ex1 = __fsub_rn(p[0], p[2]), ey1 = __fsub_rn(p[1], p[3]);
    const float ex2 = __fsub_rn(p[2], p[4]), ey2 = __fsub_rn(p[3], p[5]);
    const float e1 = __fsqrt_rn(__fadd_rn(__fmul_rn(ex1, ex1), __fmul_rn(ey1, ey1)));
    const float e2 = __fsqrt_rn(__fadd_rn(__fmul_rn(ex2, ex2), __fmul_rn(ey2, ey2)));
    const float dx1 = __fsub_rn(p[2], p[0]), dy1 = __fsub_rn(p[3], p[1]);   // pt2 - pt1
    const float dx2 = __fsub_rn(p[6], p[0]), dy2 = __fsub_rn(p[7], p[1]);   // pt4 - pt1
    const float mx = e2 > e1 ? e2 : e1, mn = e2 < e1 ? e2 : e1;
    RBox r;
    if (__fdiv_rn(mx, mn) < 1.15f) {
        r.w = mx;
        r.h = mn;
        const double a1 = norm_angle(np_atan2(dy1, dx1)), a2 = norm_angle(np_atan2(dy2, dx2));
        r.a = abs_angle_greater(a1, a2, dx1, dy1, dx2, dy2) ? a2 : a1;
    } else if (e1 > e2) {
        r.w = e1;
        r.h = e2;
        r.a = norm_angle(np_atan2(dy1, dx1));
    } else if (e2 >= e1) {
        r.w = e2;
        r.h = e1;
        r.a = norm_angle(np_atan2(dy2, dx2));
    } else {                                       // a NaN edge: neither branch, final_angle = norm_angle(0)
        r.w = r.h = 0.0;
        r.a = norm_angle(0.0);
    }
    r.x = __ddiv_rn((double)__fadd_rn(p[0], p[4]), 2.0);
    r.y = __ddiv_rn((double)__fadd_rn(p[1], p[5]), 2.0);
    return r;
}

__global__ void __launch_bounds__(kEvalThreads)
poly2rbox_v3_kernel(const double *__restrict__ quad, int n, double *__restrict__ out)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const RBox r = poly2rbox_v3(quad + (size_t)i * 8);
        double *o = out + (size_t)i * 5;
        o[0] = r.x; o[1] = r.y; o[2] = r.w; o[3] = r.h; o[4] = r.a;
    }
}

// angle_dif of every matched position: abs(v3(det) - v3(gt[jmax])) * 57.32 (mAOE_evaluation.py:158-166); NaN unmatched
__global__ void __launch_bounds__(kEvalThreads)
aoe_angle_kernel(const int32_t *__restrict__ jm, const int32_t *__restrict__ order, const double *__restrict__ det_quad,
                 const double *__restrict__ gq, int nd, double *__restrict__ angle_dif)
{
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < nd; p += gridDim.x * blockDim.x) {
        const int j = jm[p];
        double v = __longlong_as_double(0x7ff8000000000000ll);
        if (j >= 0) {
            const double a_det = poly2rbox_v3(det_quad + (size_t)order[p] * 8).a;
            const double a_gt = poly2rbox_v3(gq + (size_t)j * 8).a;
            v = __dmul_rn(fabs(__dsub_rn(a_det, a_gt)), 57.32);
        }
        angle_dif[p] = v;
    }
}

// per class, one warp: count of matched positions and aoe = (left-to-right running sum of their angle_dif) / count, the
// plain loop of mAOE_evaluation.py:192-197.  Lanes load 32 positions at a time; the adds run in rank order on every lane.
__global__ void __launch_bounds__(kEvalThreads)
aoe_class_kernel(const double *__restrict__ angle_dif, const int32_t *__restrict__ jm, const int64_t *__restrict__ cls_off,
                 int ncls, int64_t *__restrict__ count, double *__restrict__ aoe)
{
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (c >= ncls) return;
    const int64_t a = cls_off[c], b = cls_off[c + 1];
    double sum = 0.0;
    long long n = 0;
    for (int64_t base = a; base < b; base += 32) {
        const int64_t k = base + lane;
        const bool m = k < b && jm[k] >= 0;
        const double v = m ? angle_dif[k] : 0.0;
        unsigned mask = __ballot_sync(0xffffffffu, m);
        n += __popc(mask);
        while (mask) {
            const int src = __ffs(mask) - 1;
            mask &= mask - 1;
            sum = __dadd_rn(sum, __shfl_sync(0xffffffffu, v, src));
        }
    }
    if (lane == 0) {
        count[c] = n;
        aoe[c] = __ddiv_rn(sum, (double)n);   // 0 / 0 = NaN for a class without a match
    }
}

// The front both evaluations share.  Detections ranked by class, then score (order_out, cls_off_out; ckey2 = class key of
// each position), ground truth in (class, image) bucket order (gq), and per position the target jm of
// eval_match_kernel<kVoc>.  With kVoc also the difficult flags, npos per class and the claims (status, claim, npos).
struct EvalFront {
    uint32_t *ckey2 = nullptr;
    int32_t *jm = nullptr, *claim = nullptr;
    uint8_t *status = nullptr, *tmp = nullptr;   // tmp: at least the `min_tmp` bytes asked for, free after the front
    double *gq = nullptr;
    unsigned long long *npos = nullptr;
};

template <bool kVoc>
int eval_front(Scratch &S, cudaStream_t st, const char *who, const int32_t *det_cls, const int32_t *det_img,
               const double *det_score, const double *det_quad, int nd, const int32_t *gt_cls, const int32_t *gt_img,
               const double *gt_quad, const uint8_t *gt_difficult, int ng, int ncls, int nimg, double ovthresh,
               size_t min_tmp, int32_t *order_out, int64_t *cls_off_out, EvalFront &F)
{
    const uint32_t none = (uint32_t)ncls * (uint32_t)nimg;
    const int cbits = key_bits((uint64_t)ncls), sbits = key_bits((uint64_t)none);
    const int T = kEvalThreads, GD = grid_for((size_t)nd, T), GG = grid_for((size_t)ng, T);

    uint64_t *skey = S.get<uint64_t>(nd), *skey2 = S.get<uint64_t>(nd);
    int32_t *iota = S.get<int32_t>(nd), *by_score = S.get<int32_t>(nd), *dpos = S.get<int32_t>(nd);
    uint32_t *ckey = S.get<uint32_t>(nd);
    F.ckey2 = S.get<uint32_t>(nd);
    uint32_t *dseg = S.get<uint32_t>(nd), *dseg2 = S.get<uint32_t>(nd);
    F.jm = S.get<int32_t>(nd);
    uint32_t *gseg = S.get<uint32_t>(ng), *gseg2 = S.get<uint32_t>(ng);
    int32_t *giota = S.get<int32_t>(ng), *gorder = S.get<int32_t>(ng);
    F.gq = S.get<double>((size_t)ng * 8);
    double4 *gbox = S.get<double4>(ng);
    uint8_t *gdiff = nullptr;
    if (kVoc) {
        F.status = S.get<uint8_t>(nd);
        F.claim = S.get<int32_t>(ng);
        gdiff = S.get<uint8_t>(ng);
        F.npos = S.get<unsigned long long>(ncls);
    }
    if (!gbox || (kVoc && !F.npos)) return fail(ORP_ECUDA, "%s: scratch allocation failed", who);
    size_t tb1 = 0, tb2 = 0, tb3 = 0, tb4 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb1, skey, skey2, iota, by_score, nd, 0, 64, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb2, ckey, F.ckey2, by_score, order_out, nd, 0, cbits, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb3, dseg, dseg2, iota, dpos, nd, 0, sbits, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb4, gseg, gseg2, giota, gorder, ng, 0, sbits, st);
    size_t tb = min_tmp;
    for (size_t v : {tb1, tb2, tb3, tb4}) tb = tb > v ? tb : v;
    F.tmp = S.get<uint8_t>(tb);
    if (!F.tmp) return fail(ORP_ECUDA, "%s: scratch allocation failed", who);
    uint8_t *tmp = F.tmp;

    if (kVoc) ORP_CUDA(cudaMemsetAsync(F.npos, 0, sizeof(unsigned long long) * (size_t)(ncls ? ncls : 1), st));
    if (ng > 0) {
        eval_gt_seg_kernel<<<GG, T, 0, st>>>(gt_cls, gt_img, ng, ncls, nimg, gseg, giota);
        ORP_LAUNCHED();
        ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb4, gseg, gseg2, giota, gorder, ng, 0, sbits, st));
        count_launches(1);
        eval_gt_gather_kernel<kVoc><<<GG, T, 0, st>>>(gt_quad, gt_difficult, gt_cls, gorder, gseg2, ng, ncls, nimg, F.gq,
                                                      gbox, gdiff, F.npos, F.claim);
        ORP_LAUNCHED();
    }
    if (nd > 0) {
        eval_det_prep_kernel<<<GD, T, 0, st>>>(det_score, nd, skey, iota);
        ORP_LAUNCHED();
        ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb1, skey, skey2, iota, by_score, nd, 0, 64, st));
        count_launches(1);
        eval_class_key_kernel<<<GD, T, 0, st>>>(det_cls, by_score, nd, ncls, ckey);
        ORP_LAUNCHED();
        ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb2, ckey, F.ckey2, by_score, order_out, nd, 0, cbits, st));
        count_launches(1);
    }
    eval_class_offsets_kernel<<<grid_for((size_t)ncls + 1, T), T, 0, st>>>(F.ckey2, nd, ncls, cls_off_out);
    ORP_LAUNCHED();
    if (nd > 0) {
        eval_det_seg_kernel<<<GD, T, 0, st>>>(det_img, order_out, F.ckey2, nd, ncls, nimg, dseg, iota);
        ORP_LAUNCHED();
        ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb3, dseg, dseg2, iota, dpos, nd, 0, sbits, st));
        count_launches(1);
        eval_match_kernel<kVoc><<<ceil_div(nd, T), T, 0, st>>>(dseg2, dpos, order_out, det_quad, nd, gseg2, F.gq, gbox,
                                                               gdiff, ng, none, ovthresh, F.claim, F.jm, F.status);
        ORP_LAUNCHED();
    }
    return ORP_OK;
}

}  // namespace
}  // namespace orp

using namespace orp;

extern "C" int orp_dota_eval_task1(const int32_t *det_cls, const int32_t *det_img, const double *det_score,
                                   const double *det_quad, int nd, const int32_t *gt_cls, const int32_t *gt_img,
                                   const double *gt_quad, const uint8_t *gt_difficult, int ng, int ncls, int nimg,
                                   double ovthresh, int use_07_metric, const double *thresholds11, int64_t *npos_out,
                                   int64_t *cls_off_out, int32_t *order_out, double *rec_out, double *prec_out,
                                   double *ap_out, void *stream)
{
    if (nd < 0 || ng < 0 || ncls < 0 || nimg < 0 || (long long)ncls * nimg >= (long long)INT32_MAX ||
        (nd > 0 && (!det_cls || !det_img || !det_score || !det_quad || !order_out || !rec_out || !prec_out)) ||
        (ng > 0 && (!gt_cls || !gt_img || !gt_quad || !gt_difficult)) ||
        (ncls > 0 && (!npos_out || !ap_out)) || !cls_off_out || (use_07_metric && !thresholds11))
        return fail(ORP_EINVAL, "orp_dota_eval_task1: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Thresholds thr{};
    if (use_07_metric) memcpy(thr.t, thresholds11, sizeof(thr.t));
    const int T = kEvalThreads, GD = grid_for((size_t)nd, T);

    Scratch S(st);
    unsigned long long *tpfp = S.get<unsigned long long>(nd), *cum = S.get<unsigned long long>(nd);
    if (!cum) return fail(ORP_ECUDA, "orp_dota_eval_task1: scratch allocation failed");
    size_t tb5 = 0;
    cub::DeviceScan::InclusiveSum(nullptr, tb5, tpfp, cum, nd, st);
    EvalFront F;
    rc = eval_front<true>(S, st, "orp_dota_eval_task1", det_cls, det_img, det_score, det_quad, nd, gt_cls, gt_img, gt_quad,
                          gt_difficult, ng, ncls, nimg, ovthresh, tb5, order_out, cls_off_out, F);
    if (rc) return rc;
    if (nd > 0) {
        eval_tpfp_kernel<<<GD, T, 0, st>>>(F.status, F.jm, F.claim, nd, tpfp);
        ORP_LAUNCHED();
        ORP_CUDA(cub::DeviceScan::InclusiveSum(F.tmp, tb5, tpfp, cum, nd, st));
        count_launches(1);
        eval_pr_kernel<<<GD, T, 0, st>>>(cum, F.ckey2, cls_off_out, F.npos, nd, ncls, rec_out, prec_out);
        ORP_LAUNCHED();
    }
    if (ncls > 0) {
        eval_ap_kernel<<<ncls, T, 0, st>>>(rec_out, prec_out, cls_off_out, use_07_metric, thr, ap_out);
        ORP_LAUNCHED();
        ORP_CUDA(cudaMemcpyAsync(npos_out, F.npos, sizeof(int64_t) * (size_t)ncls, cudaMemcpyDeviceToDevice, st));
    }
    return ORP_OK;
}

extern "C" int orp_dota_eval_aoe(const int32_t *det_cls, const int32_t *det_img, const double *det_score,
                                 const double *det_quad, int nd, const int32_t *gt_cls, const int32_t *gt_img,
                                 const double *gt_quad, int ng, int ncls, int nimg, double ovthresh, int64_t *cls_off_out,
                                 int32_t *order_out, double *angle_dif_out, int64_t *count_out, double *aoe_out,
                                 void *stream)
{
    if (nd < 0 || ng < 0 || ncls < 0 || nimg < 0 || (long long)ncls * nimg >= (long long)INT32_MAX ||
        (nd > 0 && (!det_cls || !det_img || !det_score || !det_quad || !order_out || !angle_dif_out)) ||
        (ng > 0 && (!gt_cls || !gt_img || !gt_quad)) || (ncls > 0 && (!count_out || !aoe_out)) || !cls_off_out)
        return fail(ORP_EINVAL, "orp_dota_eval_aoe: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int T = kEvalThreads;
    Scratch S(st);
    EvalFront F;
    rc = eval_front<false>(S, st, "orp_dota_eval_aoe", det_cls, det_img, det_score, det_quad, nd, gt_cls, gt_img, gt_quad,
                           nullptr, ng, ncls, nimg, ovthresh, 0, order_out, cls_off_out, F);
    if (rc) return rc;
    if (nd > 0) {
        aoe_angle_kernel<<<grid_for((size_t)nd, T), T, 0, st>>>(F.jm, order_out, det_quad, F.gq, nd, angle_dif_out);
        ORP_LAUNCHED();
    }
    if (ncls > 0) {
        aoe_class_kernel<<<ceil_div((long long)ncls * 32, T), T, 0, st>>>(angle_dif_out, F.jm, cls_off_out, ncls, count_out,
                                                                           aoe_out);
        ORP_LAUNCHED();
    }
    return ORP_OK;
}

extern "C" int orp_poly2rbox_v3(const double *quad, int n, double *out, void *stream)
{
    if (n < 0 || (n > 0 && (!quad || !out))) return fail(ORP_EINVAL, "orp_poly2rbox_v3: bad arguments");
    if (n == 0) return ORP_OK;
    int rc = ensure_device();
    if (rc) return rc;
    poly2rbox_v3_kernel<<<grid_for((size_t)n, kEvalThreads), kEvalThreads, 0, static_cast<cudaStream_t>(stream)>>>(quad, n, out);
    ORP_LAUNCHED();
    return ORP_OK;
}
