// merge.cu - DOTA ResultMerge over the packed detection buffer (orp_result_merge).
//
// Replaces the text stage between the detector's gather and the Task1 evaluation: the Task1 writer of
// tools/parse_pkl/parse_pkl_mege_results_for_dota_evaluation.py:93-192 and mergesingle / poly2origpoly / nmsbynamedict of
// DOTA_devkit/ResultMerge_multi_process.py:156-223, which print every detection, parse it back and run a Python NMS per
// original image and class.  Here the rows never leave the device:
//
//   count    a warp per dataset tile checks the tile's slot, count and metadata and counts the rows whose label is a class
//   scan     exclusive sum of the tile counts -> the row number of each tile's first detection: rows are numbered in
//            dataset tile order, then in-tile order - the order of the text path's lines within a class
//   restore  a warp per tile compacts its rows in order (ballot + popc), restores the quadrilateral to image coordinates in
//            fp64 as poly2origpoly (:173-180) does, and reduces per (class, image) segment the smallest finite x and y and
//            the smallest row number with order-preserving integer atomicMin
//   rows     fp32 NMS rows: every segment translated, in fp64, to floor(min x), floor(min y) of its own boxes (IoU is
//            translation invariant; the cast then costs ~1e-5 px instead of ~1e-3 px); rows past the last detection are
//            NaN boxes, which the NMS keeps without comparing and the ordering drops
//   nms      run_nms: ORP_NMS_EXACT64, score descending, segment = class * nimg + image
//   order    one stable radix sort of the keep list by (class, first row of the segment): the merged files' order - class,
//            then original image by first appearance among the class's rows, then score descending (ties in row order)
#include <cub/cub.cuh>

#include "common.cuh"

namespace orp {
namespace {

constexpr int kMergeThreads = 256;
constexpr int kRowFloats = 28;          // reppoints(18) | box(8) | score | label
constexpr int kBoxCol = 18, kScoreCol = 26, kLabelCol = 27;

// double -> unsigned key whose ascending order is the ascending order of the finite doubles, and back
__device__ __forceinline__ unsigned long long f64_orderable(double v)
{
    const unsigned long long u = (unsigned long long)__double_as_longlong(v);
    return (u >> 63) ? ~u : (u | (1ull << 63));
}
__device__ __forceinline__ double f64_from_orderable(unsigned long long k)
{
    return __longlong_as_double((long long)((k >> 63) ? (k ^ (1ull << 63)) : ~k));
}

// the class of a row, or -1: labels travel as fp32 and must be integers in [0, ncls)
__device__ __forceinline__ int row_class(float label, int ncls)
{
    return (label >= 0.0f && label < (float)ncls && label == floorf(label)) ? (int)label : -1;
}

// the slot's detection count (row `cap`, column 0), or -1 when it is not an integer in [0, cap]
__device__ __forceinline__ int slot_count(const float *__restrict__ packed, int slot, int cap)
{
    const float c = packed[((size_t)slot * (cap + 1) + cap) * kRowFloats];
    return (c >= 0.0f && c <= (float)cap && c == floorf(c)) ? (int)c : -1;
}

__global__ void __launch_bounds__(kMergeThreads)
merge_count_kernel(const float *__restrict__ packed, int S, int cap, const int32_t *__restrict__ tile_slot,
                   const double *__restrict__ tile_rate, const int32_t *__restrict__ tile_img, int Tn, int ncls, int nimg,
                   int32_t *__restrict__ tile_cnt, int32_t *__restrict__ status)
{
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < Tn; i += warps) {
        const int slot = tile_slot[i];
        int cnt = 0;
        if (slot >= 0) {
            const double rate = tile_rate[i];
            const int img = tile_img[i];
            int c = slot < S ? slot_count(packed, slot, cap) : 0;
            // the rest of the count row is zero padding (orp_pack_detections): anything else there means the buffer is not
            // in the packed layout, e.g. its count row was cut off and a detection row is read in its place
            const bool stray = slot < S && lane >= 1 && lane < kRowFloats &&
                               packed[((size_t)slot * (cap + 1) + cap) * kRowFloats + lane] != 0.0f;
            if (__any_sync(0xffffffffu, stray)) c = -1;
            if (slot >= S || !(rate > 0.0) || isinf(rate) || img < 0 || img >= nimg) {
                if (lane == 0) atomicOr(status, ORP_MERGE_BAD_TILE);
            } else if (c < 0) {
                if (lane == 0) atomicOr(status, ORP_MERGE_BAD_COUNT);
            } else {
                const float *rows = packed + (size_t)slot * (cap + 1) * kRowFloats;
                for (int r = lane; r < c; r += 32) cnt += row_class(rows[(size_t)r * kRowFloats + kLabelCol], ncls) >= 0;
                for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
            }
        }
        if (lane == 0) tile_cnt[i] = cnt;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) tile_cnt[Tn] = 0;   // the scan's last element: the total lands there
}

__global__ void __launch_bounds__(kMergeThreads)
merge_restore_kernel(const float *__restrict__ packed, int cap, const int32_t *__restrict__ tile_slot,
                     const int32_t *__restrict__ tile_xy, const double *__restrict__ tile_rate,
                     const int32_t *__restrict__ tile_img, int Tn, int ncls, int nimg, const int32_t *__restrict__ tile_cnt,
                     const int32_t *__restrict__ tile_off, int max_rows, double *__restrict__ quad, double *__restrict__ score,
                     int32_t *__restrict__ seg, unsigned long long *__restrict__ seg_ox,
                     unsigned long long *__restrict__ seg_oy, int32_t *__restrict__ seg_first, int32_t *__restrict__ status)
{
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < Tn; i += warps) {
        if (tile_cnt[i] == 0) continue;                           // skipped, refused or without a labelled row
        const int slot = tile_slot[i], img = tile_img[i];
        const int c = slot_count(packed, slot, cap);
        const double ox = (double)tile_xy[2 * i], oy = (double)tile_xy[2 * i + 1], rate = tile_rate[i];
        const float *rows = packed + (size_t)slot * (cap + 1) * kRowFloats;
        int base = tile_off[i];
        for (int r0 = 0; r0 < c; r0 += 32) {
            const int r = r0 + lane;
            const float *row = rows + (size_t)r * kRowFloats;
            const int cls = r < c ? row_class(row[kLabelCol], ncls) : -1;
            const unsigned mask = __ballot_sync(0xffffffffu, cls >= 0);
            const int pos = base + __popc(mask & ((1u << lane) - 1u));
            base += __popc(mask);
            if (cls < 0) continue;
            if (pos >= max_rows) { atomicOr(status, ORP_MERGE_ROWS_OVERFLOW); continue; }
            // poly2origpoly: (p + x) / rate in IEEE double, the two operations rounded on their own
            double xmin = INFINITY, ymin = INFINITY;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const double x = __ddiv_rn(__dadd_rn((double)row[kBoxCol + 2 * k], ox), rate);
                const double y = __ddiv_rn(__dadd_rn((double)row[kBoxCol + 2 * k + 1], oy), rate);
                quad[(size_t)pos * 8 + 2 * k] = x;
                quad[(size_t)pos * 8 + 2 * k + 1] = y;
                if (isfinite(x) && x < xmin) xmin = x;
                if (isfinite(y) && y < ymin) ymin = y;
            }
            score[pos] = (double)row[kScoreCol];
            const int s = cls * nimg + img;
            seg[pos] = s;
            if (xmin < INFINITY) atomicMin(&seg_ox[s], f64_orderable(xmin));
            if (ymin < INFINITY) atomicMin(&seg_oy[s], f64_orderable(ymin));
            atomicMin(&seg_first[s], pos);
        }
    }
}

// the NMS input: [max_rows, 9] fp32 rows about their segment's origin, and the segment ids
__global__ void __launch_bounds__(kMergeThreads)
merge_rows_kernel(const double *__restrict__ quad, const double *__restrict__ score, const int32_t *__restrict__ seg,
                  const unsigned long long *__restrict__ seg_ox, const unsigned long long *__restrict__ seg_oy,
                  const int32_t *__restrict__ total, int max_rows, float *__restrict__ rows9, int32_t *__restrict__ segs,
                  int32_t *__restrict__ status)
{
    const int n = min(*total, max_rows);
    if (blockIdx.x == 0 && threadIdx.x == 0 && *total > max_rows) atomicOr(status, ORP_MERGE_ROWS_OVERFLOW);
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < max_rows; r += gridDim.x * blockDim.x) {
        float *o = rows9 + (size_t)r * 9;
        if (r >= n) {
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = __int_as_float(0x7fc00000);
            o[8] = -INFINITY;
            segs[r] = 0;
            continue;
        }
        const int s = seg[r];
        // a segment without a finite coordinate keeps the origin 0
        const unsigned long long kx = seg_ox[s], ky = seg_oy[s];
        const double fx = kx == ~0ull ? 0.0 : floor(f64_from_orderable(kx));
        const double fy = ky == ~0ull ? 0.0 : floor(f64_from_orderable(ky));
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            o[2 * k] = __double2float_rn(__dsub_rn(quad[(size_t)r * 8 + 2 * k], fx));
            o[2 * k + 1] = __double2float_rn(__dsub_rn(quad[(size_t)r * 8 + 2 * k + 1], fy));
        }
        o[8] = (float)score[r];                                   // exact: the score was widened from fp32
        segs[r] = s;
    }
}

// sort key of every position of the keep list: (class : first row of the segment); positions past the list and the
// padding rows get the key of class `ncls`, after every class
__global__ void __launch_bounds__(kMergeThreads)
merge_keys_kernel(const int64_t *__restrict__ keep, const int32_t *__restrict__ num_keep, const int32_t *__restrict__ total,
                  const int32_t *__restrict__ seg, const int32_t *__restrict__ seg_first, int max_rows, int ncls, int nimg,
                  uint64_t *__restrict__ key, int32_t *__restrict__ val)
{
    const int n = min(*total, max_rows), nk = *num_keep;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < max_rows; k += gridDim.x * blockDim.x) {
        uint64_t v = ((uint64_t)ncls << 32) | 0xFFFFFFFFull;
        int r = 0;
        if (k < nk && (r = (int)keep[k]) < n) {
            const int s = seg[r];
            v = ((uint64_t)(s / nimg) << 32) | (uint32_t)seg_first[s];
        }
        key[k] = v;
        val[k] = r;
    }
}

__device__ __forceinline__ int lower_bound_u64(const uint64_t *a, int n, uint64_t v)
{
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(kMergeThreads)
merge_offsets_kernel(const uint64_t *__restrict__ key, int max_rows, int ncls, int64_t *__restrict__ cls_off,
                     int32_t *__restrict__ count)
{
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= ncls; c += gridDim.x * blockDim.x) {
        const int off = lower_bound_u64(key, max_rows, (uint64_t)c << 32);
        cls_off[c] = off;
        if (c == ncls) *count = off;
    }
}

__global__ void __launch_bounds__(kMergeThreads)
merge_gather_kernel(const uint64_t *__restrict__ key, const int32_t *__restrict__ val, const double *__restrict__ quad,
                    const double *__restrict__ score, const int32_t *__restrict__ seg, int max_rows, int ncls, int nimg,
                    int32_t *__restrict__ out_cls, int32_t *__restrict__ out_img, double *__restrict__ out_score,
                    double *__restrict__ out_quad, int32_t *__restrict__ out_row)
{
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < max_rows; k += gridDim.x * blockDim.x) {
        if ((key[k] >> 32) >= (uint64_t)ncls) continue;
        const int r = val[k], s = seg[r];
        out_cls[k] = s / nimg;
        out_img[k] = s % nimg;
        out_score[k] = score[r];
        out_row[k] = r;
#pragma unroll
        for (int j = 0; j < 8; ++j) out_quad[(size_t)k * 8 + j] = quad[(size_t)r * 8 + j];
    }
}

}  // namespace
}  // namespace orp

using namespace orp;

extern "C" int orp_result_merge(const float *packed, int S, int cap, const int32_t *tile_slot, const int32_t *tile_xy,
                                const double *tile_rate, const int32_t *tile_img, int Tn, int ncls, int nimg, double thresh,
                                int union_mode, int max_rows, int32_t *count_out, int64_t *cls_off_out, int32_t *cls_out,
                                int32_t *img_out, double *score_out, double *quad_out, int32_t *src_row_out,
                                int32_t *status_out, void *stream)
{
    if (S < 0 || cap < 1 || Tn < 0 || ncls < 1 || nimg < 1 || max_rows < 0 ||
        (long long)ncls * nimg >= (long long)INT32_MAX || (long long)S * ((long long)cap + 1) >= (long long)INT32_MAX ||
        (long long)Tn * cap >= (long long)INT32_MAX)   // rows are numbered in int32, and a slot may be selected more than once
        return fail(ORP_EINVAL, "orp_result_merge: sizes out of range");
    if (!count_out || !cls_off_out || !status_out || (S > 0 && !packed) ||
        (Tn > 0 && (!tile_slot || !tile_xy || !tile_rate || !tile_img)) ||
        (max_rows > 0 && (!cls_out || !img_out || !score_out || !quad_out || !src_row_out)))
        return fail(ORP_EINVAL, "orp_result_merge: null pointer");
    if (union_mode != ORP_UNION_NAN_SUPPRESSES && union_mode != ORP_UNION_NAN_SUPPRESSES_ALL)
        return fail(ORP_EINVAL, "orp_result_merge: union_mode must be ORP_UNION_NAN_SUPPRESSES or ORP_UNION_NAN_SUPPRESSES_ALL");
    if (!(thresh == thresh)) return fail(ORP_EINVAL, "orp_result_merge: thresh is NaN");
    int rc = ensure_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int T = kMergeThreads, nseg = ncls * nimg;
    const int GT = grid_for((size_t)Tn * 32, T), GR = grid_for((size_t)max_rows, T);
    const int kbits = 32 + key_bits((uint64_t)ncls);

    Scratch sc(st);
    int32_t *tile_cnt = sc.get<int32_t>((size_t)Tn + 1), *tile_off = sc.get<int32_t>((size_t)Tn + 1);
    double *quad = sc.get<double>((size_t)max_rows * 8), *score = sc.get<double>(max_rows);
    int32_t *seg = sc.get<int32_t>(max_rows), *segs = sc.get<int32_t>(max_rows);
    unsigned long long *seg_ox = sc.get<unsigned long long>((size_t)nseg * 2), *seg_oy = seg_ox ? seg_ox + nseg : nullptr;
    int32_t *seg_first = sc.get<int32_t>(nseg);
    float *rows9 = sc.get<float>((size_t)max_rows * 9);
    int64_t *keep = sc.get<int64_t>(max_rows);
    int32_t *num_keep = sc.get<int32_t>(1);
    uint64_t *key = sc.get<uint64_t>(max_rows), *key2 = sc.get<uint64_t>(max_rows);
    int32_t *val = sc.get<int32_t>(max_rows), *val2 = sc.get<int32_t>(max_rows);
    size_t tb1 = 0, tb2 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb1, tile_cnt, tile_off, Tn + 1, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb2, key, key2, val, val2, max_rows, 0, kbits, st);
    uint8_t *tmp = sc.get<uint8_t>(tb1 > tb2 ? tb1 : tb2);
    if (!tmp || !val2 || !key2 || !num_keep || !keep || !rows9 || !seg_first || !seg_ox || !segs || !score || !quad || !tile_off)
        return fail(ORP_ECUDA, "orp_result_merge: scratch allocation failed");

    ORP_CUDA(cudaMemsetAsync(status_out, 0, sizeof(int32_t), st));
    ORP_CUDA(cudaMemsetAsync(count_out, 0, sizeof(int32_t), st));
    ORP_CUDA(cudaMemsetAsync(cls_off_out, 0, sizeof(int64_t) * ((size_t)ncls + 1), st));
    ORP_CUDA(cudaMemsetAsync(seg_ox, 0xFF, sizeof(unsigned long long) * (size_t)nseg * 2, st));
    ORP_CUDA(cudaMemsetAsync(seg_first, 0x7F, sizeof(int32_t) * (size_t)nseg, st));

    merge_count_kernel<<<GT, T, 0, st>>>(packed, S, cap, tile_slot, tile_rate, tile_img, Tn, ncls, nimg, tile_cnt, status_out);
    ORP_LAUNCHED();
    ORP_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb1, tile_cnt, tile_off, Tn + 1, st));
    count_launches(1);
    if (Tn > 0) {
        merge_restore_kernel<<<GT, T, 0, st>>>(packed, cap, tile_slot, tile_xy, tile_rate, tile_img, Tn, ncls, nimg, tile_cnt,
                                               tile_off, max_rows, quad, score, seg, seg_ox, seg_oy, seg_first, status_out);
        ORP_LAUNCHED();
    }
    merge_rows_kernel<<<GR, T, 0, st>>>(quad, score, seg, seg_ox, seg_oy, tile_off + Tn, max_rows, rows9, segs, status_out);
    ORP_LAUNCHED();
    if (max_rows == 0) return ORP_OK;

    rc = run_nms(rows9, segs, max_rows, thresh, ORP_NMS_EXACT64, union_mode, ORP_ORDER_SCORE_DESC, keep, num_keep, st, nullptr,
                 false, nseg, nullptr);
    if (rc) return rc;

    merge_keys_kernel<<<GR, T, 0, st>>>(keep, num_keep, tile_off + Tn, seg, seg_first, max_rows, ncls, nimg, key, val);
    ORP_LAUNCHED();
    ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb2, key, key2, val, val2, max_rows, 0, kbits, st));
    count_launches((kbits + 7) / 8);
    merge_offsets_kernel<<<grid_for((size_t)ncls + 1, T), T, 0, st>>>(key2, max_rows, ncls, cls_off_out, count_out);
    ORP_LAUNCHED();
    merge_gather_kernel<<<GR, T, 0, st>>>(key2, val2, quad, score, seg, max_rows, ncls, nimg, cls_out, img_out, score_out,
                                          quad_out, src_row_out);
    ORP_LAUNCHED();
    return ORP_OK;
}
