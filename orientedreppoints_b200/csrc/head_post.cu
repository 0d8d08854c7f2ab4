// head_post.cu - OrientedRepPointsHead.get_bboxes + multiclass_rnms as a device-resident pipeline
// (SURVEY.md section 8 rows a7, a9): no host round trip until the caller reads the counts.
//
// Replaces mmdet/models/anchor_heads/orientedreppoints_head.py:673-779 (per level: sigmoid, max-over-class
// top-k(nms_pre), (dy,dx)->(x,y), minaerarect, *stride + centre) and
// mmdet/core/post_processing/bbox_nms.py:93-182 (score threshold, class-aware rnms, max_per_img) for a
// whole batch at once:
//   1. maxscore   levels with H*W > nms_pre: key = (segment, ~order(max_c sigmoid)) -> ONE radix sort
//                 (stable: equal scores keep ascending location order)
//   2. decode     one thread per (image, candidate slot): 18 offsets -> hull -> min-area rectangle ->
//                 box*stride + centre, reppoints, 15 sigmoid scores; writes the NMS input rows
//                 (box, score) for every class with segment id = image*C + class; rows at or below the
//                 score threshold are poisoned (NaN) so the NMS sweep skips them
//   3. nms        segmented rotated NMS (nms.cu), survivor flags by candidate index
//   4. select     per image: survivors in candidate order, or - when more than max_per_img survive - the
//                 max_per_img best by score; ONE radix sort on (image, mode key, index)
//   5. gather     [B, max_per_img, 27] rows (reppoints | box | score), labels, counts
//
// The same pipeline serves multi-view test-time augmentation (orp_head_postprocess_aug), which replaces
// OrientedRepPointsDetector.aug_test's post-processing (mmdet/models/detectors/orientedreppoints_detector.py:48-144:
// get_bboxes(rescale=False, nms=False) per view, rbox_mapping_back, torch.cat, ONE multiclass_rnms) for V views of B
// images.  The level table holds V * nlevels entries, view-major, so an image's candidates are ordered as torch.cat
// over the views orders them, and the NMS segment stays image * C + class: the views of an image share segments and a
// box of the flipped view suppresses its twin of the identity view.  The decode maps every box back into the image
// frame, in the arithmetic of that eager code rather than simple_test's (each step one fp32 rounding):
//   box = rect * stride + centre                       (no division here: rescale=False, head :748-749)
//   flipped view:  x = (w - x) - 1 on the four vertices, w = float(img_shape[1])            (:53-61)
//   every view:    box * (1.0f / scale_factor)         (:96; the eager code divides a CUDA tensor by a Python float,
//                  which torch evaluates as a product with the fp32 reciprocal - not x / scale_factor, the division by a
//                  device tensor that simple_test's rescale performs; the two differ in the last bit for a factor that
//                  is not a power of two)
// and, when the caller keeps the first view's frame (rescale=False, :139-141), the 8 box values of the selected rows are
// multiplied by out_scale[image] in the gather.  These rows carry no reppoints: columns 0..17 are zero.
#include <cub/cub.cuh>

#include "common.cuh"
#include "minrect.cuh"

namespace orp {
namespace {

constexpr int kMaxLevels = 8;       // levels of one view
constexpr int kMaxEntries = 80;     // (view, level) entries of a call; the table travels as a kernel argument (< 4 KB)

struct Levels {                 // one entry per (view, level), view-major
    const float *cls[kMaxEntries], *ref[kMaxEntries];
    int H[kMaxEntries], W[kMaxEntries], stride[kMaxEntries];
    int slot0[kMaxEntries];     // first candidate slot of the entry inside an image; it holds min(H*W, nms_pre) slots
    int sort0[kMaxEntries];     // offset of (entry, image 0) inside the sort arrays, -1 if the entry skips the top-k sort
    int nent, per_view, B, C, S;    // entries, levels per view, S = slots per image
};
static_assert(sizeof(Levels) <= 4000, "the level table is a kernel argument");

__device__ __forceinline__ float sigmoidf_ref(float x) { return 1.0f / (1.0f + expf(-x)); }   // == torch.sigmoid (fp32)

__global__ void __launch_bounds__(256)
maxscore_kernel(const __grid_constant__ Levels L, int lev, uint64_t *__restrict__ keys, int32_t *__restrict__ vals)
{
    const int HW = L.H[lev] * L.W[lev];
    const size_t total = (size_t)L.B * HW;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / HW), loc = (int)(i - (size_t)b * HW);
        const float *c = L.cls[lev] + i * L.C;
        float m = sigmoidf_ref(c[0]);
        for (int k = 1; k < L.C; ++k) m = fmaxf(m, sigmoidf_ref(c[k]));
        const size_t o = (size_t)L.sort0[lev] + i;
        // ascending sort on (segment start offset, descending score); stable -> ascending location on ties
        keys[o] = ((uint64_t)(uint32_t)(L.sort0[lev] + b * HW) << 32) | (uint64_t)(~orderable(m));
        vals[o] = loc;
    }
}

struct DecodeOut {
    float *dets;        // [B*S*C, 9]
    int32_t *segs;      // [B*S*C]
    uint8_t *valid;     // [B*S*C]
    float *rp;          // [B*S, 18]
    float *box;         // [B*S, 8]
};

// kAug: the multi-view mode; view_meta is device fp32 [nviews, B, 3] = flip (0 / 1), img_shape width, scale_factor
template <bool kAug>
__global__ void __launch_bounds__(128)
decode_kernel(const __grid_constant__ Levels L, const int32_t *__restrict__ sorted_vals, float score_thr,
              const float *__restrict__ scale_factor, const float *__restrict__ view_meta, DecodeOut O)
{
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= L.B * L.S) return;
    const int b = gid / L.S, slot = gid - b * L.S;
    int lev = 0;
    for (int k = 1; k < L.nent; ++k) if (slot >= L.slot0[k]) lev = k;
    const int k = slot - L.slot0[lev];
    const int HW = L.H[lev] * L.W[lev];
    const int loc = L.sort0[lev] >= 0 ? sorted_vals[(size_t)L.sort0[lev] + (size_t)b * HW + k] : k;
    const int y = loc / L.W[lev], x = loc - y * L.W[lev];
    const float st = (float)L.stride[lev];
    const float cx = (float)x * st, cy = (float)y * st;               // point_generator.py:14-22
    const float *pr = L.ref[lev] + ((size_t)b * HW + loc) * 18;
    float in[18], rect[8];
#pragma unroll
    for (int p = 0; p < 9; ++p) { in[2 * p] = pr[2 * p + 1]; in[2 * p + 1] = pr[2 * p]; }   // (dy,dx) -> (x,y), head :742-745
    mr::minrect_one(in, rect, nullptr);
    float box[8];
    if (kAug) {
        const float *m = view_meta + ((size_t)(lev / L.per_view) * L.B + b) * 3;
        const bool flip = m[0] != 0.f;
        const float w = m[1], inv = __fdiv_rn(1.0f, m[2]);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float bx = __fadd_rn(__fmul_rn(rect[2 * c], st), cx);      // head :748-749, rescale=False
            if (flip) bx = __fsub_rn(__fsub_rn(w, bx), 1.0f);          // detector :53-61
            box[2 * c] = __fmul_rn(bx, inv);                            // detector :96, see the note at the top
            box[2 * c + 1] = __fmul_rn(__fadd_rn(__fmul_rn(rect[2 * c + 1], st), cy), inv);
        }
    } else {
        const float sf = scale_factor ? scale_factor[b] : 1.0f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            box[2 * c] = __fdiv_rn(__fadd_rn(__fmul_rn(rect[2 * c], st), cx), sf);             // :748-749, :766-768
            box[2 * c + 1] = __fdiv_rn(__fadd_rn(__fmul_rn(rect[2 * c + 1], st), cy), sf);
        }
        float *rp = O.rp + (size_t)gid * 18;
#pragma unroll
        for (int p = 0; p < 9; ++p) {
            rp[2 * p] = __fdiv_rn(__fadd_rn(__fmul_rn(in[2 * p], st), cx), sf);
            rp[2 * p + 1] = __fdiv_rn(__fadd_rn(__fmul_rn(in[2 * p + 1], st), cy), sf);
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) O.box[(size_t)gid * 8 + c] = box[c];
    const float *cl = L.cls[lev] + ((size_t)b * HW + loc) * L.C;
    for (int c = 0; c < L.C; ++c) {
        const float s = sigmoidf_ref(cl[c]);
        const size_t row = (size_t)gid * L.C + c;
        const bool ok = s > score_thr;                                 // bbox_nms.py:131
        float *d = O.dets + row * 9;
        d[0] = ok ? box[0] : __int_as_float(0x7fc00000);               // NaN poisons the row for the sweep
#pragma unroll
        for (int q = 1; q < 8; ++q) d[q] = box[q];
        d[8] = s;
        O.segs[row] = b * L.C + c;
        O.valid[row] = ok ? 1 : 0;
    }
}

__global__ void __launch_bounds__(256)
count_kernel(const uint8_t *__restrict__ keep, const uint8_t *__restrict__ valid, int per_img, int B, int32_t *__restrict__ counts)
{
    __shared__ int s_cnt;
    const int b = blockIdx.y;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_img; i += gridDim.x * blockDim.x) {
        const size_t r = (size_t)b * per_img + i;
        c += (keep[r] && valid[r]) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0 && s_cnt) atomicAdd(&counts[b], s_cnt);
}

__global__ void __launch_bounds__(256)
select_keys_kernel(const uint8_t *__restrict__ keep, const uint8_t *__restrict__ valid, const float *__restrict__ dets,
                   const int32_t *__restrict__ counts, int per_img, int B, int cap, uint64_t *__restrict__ keys,
                   int32_t *__restrict__ vals)
{
    const size_t total = (size_t)B * per_img;
    for (size_t r = blockIdx.x * (size_t)blockDim.x + threadIdx.x; r < total; r += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(r / per_img), i = (int)(r - (size_t)b * per_img);
        uint64_t mid;
        if (!(keep[r] && valid[r])) mid = 0xFFFFFFFFull;
        else if (counts[b] > cap) mid = (uint64_t)(~orderable(dets[r * 9 + 8]));   // score descending (top bit clear: never 0xFFFFFFFF)
        else mid = 0;                                                                              // candidate order
        keys[r] = ((uint64_t)b << 32) | mid;        // the sort is stable: ties keep candidate order
        vals[r] = i;
    }
}

__global__ void __launch_bounds__(128)
gather_kernel(const int32_t *__restrict__ sorted_vals, const int32_t *__restrict__ counts, const float *__restrict__ dets,
              const float *__restrict__ rp, const float *__restrict__ box, const float *__restrict__ out_scale, int per_img,
              int S, int C, int cap, int B, float *__restrict__ out, int64_t *__restrict__ labels,
              int32_t *__restrict__ counts_out, const int32_t *__restrict__ nms_overflow)
{
    const int b = blockIdx.y;
    const int n = counts[b] < cap ? counts[b] : cap;
    const float os = out_scale ? out_scale[b] : 1.0f;                 // x * 1.0f is x, bit for bit
    // a candidate-list overflow inside the NMS (no host sync on this path) poisons the counts: -1 = "results invalid"
    if (blockIdx.x == 0 && threadIdx.x == 0) counts_out[b] = *nms_overflow ? -1 : n;
    for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < cap; j += gridDim.x * blockDim.x) {
        float *o = out + ((size_t)b * cap + j) * 27;
        if (j < n) {
            const int i = sorted_vals[(size_t)b * per_img + j];
            const int slot = i / C, c = i - slot * C;
            const size_t g = (size_t)b * S + slot;
#pragma unroll
            for (int q = 0; q < 18; ++q) o[q] = rp ? rp[g * 18 + q] : 0.f;      // rp == NULL: multi-view rows carry no reppoints
#pragma unroll
            for (int q = 0; q < 8; ++q) o[18 + q] = __fmul_rn(box[g * 8 + q], os);
            o[26] = dets[((size_t)b * per_img + i) * 9 + 8];
            labels[(size_t)b * cap + j] = c;
        } else {
#pragma unroll
            for (int q = 0; q < 27; ++q) o[q] = 0.f;
            labels[(size_t)b * cap + j] = -1;
        }
    }
}

// padded detections -> the all-gather payload [B, cap + 1, 28]: rows = 27 detection values | label, zero padded; row `cap`
// carries the image's count in column 0 (orientedreppoints_b200/gather.py layout) - one launch instead of a fill + 3 copies
__global__ void __launch_bounds__(256)
pack_kernel(const float *__restrict__ dets, const int64_t *__restrict__ labels, const int32_t *__restrict__ counts, int B, int cap,
            float *__restrict__ out)
{
    const size_t total = (size_t)B * (cap + 1) * 28;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int col = (int)(i % 28);
        const size_t row = i / 28;
        const int r = (int)(row % (cap + 1)), b = (int)(row / (cap + 1));
        float v = 0.f;
        if (r < cap) v = col < 27 ? dets[((size_t)b * cap + r) * 27 + col] : (float)labels[(size_t)b * cap + r];
        else if (col == 0) v = (float)counts[b];
        out[i] = v;
    }
}

// head :162-163 for all levels at once:  offset = (1 - g) * pts + g * pts - base[c]  (fp32, evaluated as written there)
struct OffsetProb { const float *pts; float *off; long long n; };
struct OffsetParams { OffsetProb p[8]; int nprob; float g; float base[18]; };
__global__ void __launch_bounds__(256)
dcn_offsets_kernel(const __grid_constant__ OffsetParams P)
{
    const OffsetProb &pr = P.p[blockIdx.y];
    const float g = P.g, og = 1.f - P.g;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < pr.n; i += (long long)gridDim.x * blockDim.x) {
        const float t = pr.pts[i];
        // no FMA contraction: the reference evaluates two products, a sum and a difference, each rounded
        pr.off[i] = __fsub_rn(__fadd_rn(__fmul_rn(og, t), __fmul_rn(g, t)), P.base[(int)(i % 18)]);
    }
}

}  // namespace
}  // namespace orp

using namespace orp;

namespace orp {
namespace {

// the one host driver of both entry points; `who` names the caller in error messages.  view_meta == NULL is the
// one-view pipeline of orp_head_postprocess (rescale by scale_factor, reppoints kept), otherwise the multi-view one.
// Every refusal comes before the first CUDA call.
int head_post(const char *who, int nviews, int nlevels, const float *const *cls, const float *const *ref, const int *H,
              const int *W, const int *stride, int B, int num_cls, int nms_pre, float score_thr, double iou_thr,
              int max_per_img, const float *scale_factor, const float *view_meta, const float *out_scale, float *dets_out,
              int64_t *labels_out, int32_t *counts_out, void *stream)
{
    if (nviews < 1 || nlevels < 1 || nlevels > kMaxLevels || !cls || !ref || !H || !W || !stride || B < 1 || num_cls < 1 ||
        !dets_out || !labels_out || !counts_out || max_per_img < 1)
        return fail(ORP_EINVAL, "%s: bad arguments", who);
    if ((long long)nviews * nlevels > kMaxEntries) return fail(ORP_EINVAL, "%s: too many (view, level) pairs", who);
    if (B * num_cls >= (1 << 20) || B >= 2048) return fail(ORP_EINVAL, "%s: batch too large", who);
    const bool aug = view_meta != nullptr;
    Levels L;
    memset(&L, 0, sizeof(L));
    L.nent = nviews * nlevels; L.per_view = nlevels; L.B = B; L.C = num_cls;
    size_t nsort = 0;
    long long S = 0;
    for (int l = 0; l < L.nent; ++l) {
        if (!cls[l] || !ref[l] || H[l] < 1 || W[l] < 1 || (long long)H[l] * W[l] >= (1 << 20))
            return fail(ORP_EINVAL, "%s: bad level", who);
        L.cls[l] = cls[l]; L.ref[l] = ref[l]; L.H[l] = H[l]; L.W[l] = W[l]; L.stride[l] = stride[l];
        const int hw = H[l] * W[l];
        const bool sorted = nms_pre > 0 && hw > nms_pre;               // head :731-740
        L.slot0[l] = (int)S;
        S += sorted ? nms_pre : hw;
        L.sort0[l] = sorted ? (int)nsort : -1;
        if (sorted) nsort += (size_t)B * hw;
        // the select keys hold a candidate index in 20 bits, the top-k keys a sort offset in 31
        if (S * num_cls >= (1 << 20)) return fail(ORP_EINVAL, "%s: too many candidates per image", who);
        if (nsort >= (1ull << 31)) return fail(ORP_EINVAL, "%s: batch too large", who);
    }
    L.S = (int)S;
    const size_t per_img = (size_t)S * num_cls, total = per_img * B;
    int rc = ensure_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Scratch Sc(st);
    uint64_t *k1 = Sc.get<uint64_t>(nsort ? nsort : 1), *k2 = Sc.get<uint64_t>(nsort ? nsort : 1);
    int32_t *v1 = Sc.get<int32_t>(nsort ? nsort : 1), *v2 = Sc.get<int32_t>(nsort ? nsort : 1);
    DecodeOut O;
    O.dets = Sc.get<float>(total * 9);
    O.segs = Sc.get<int32_t>(total);
    O.valid = Sc.get<uint8_t>(total);
    O.rp = aug ? nullptr : Sc.get<float>((size_t)B * S * 18);
    O.box = Sc.get<float>((size_t)B * S * 8);
    uint8_t *keep = Sc.get<uint8_t>(total);
    int32_t *counts = Sc.get<int32_t>(B);
    uint64_t *sk1 = Sc.get<uint64_t>(total), *sk2 = Sc.get<uint64_t>(total);
    int32_t *sv1 = Sc.get<int32_t>(total), *sv2 = Sc.get<int32_t>(total);
    size_t tb1 = 0, tb2 = 0;
    if (nsort) cub::DeviceRadixSort::SortPairs(nullptr, tb1, k1, k2, v1, v2, (int)nsort, 0, 64, st);
    const int sel_bits = 32 + key_bits((uint64_t)B - 1);              // (image << 32 | score key)
    cub::DeviceRadixSort::SortPairs(nullptr, tb2, sk1, sk2, sv1, sv2, (int)total, 0, sel_bits, st);
    uint8_t *tmp = Sc.get<uint8_t>(tb1 > tb2 ? tb1 : tb2);
    if (!tmp || !sv2 || !keep) return fail(ORP_ECUDA, "%s: scratch allocation failed", who);

    if (nsort) {
        for (int l = 0; l < L.nent; ++l)
            if (L.sort0[l] >= 0) {
                maxscore_kernel<<<grid_for((size_t)B * H[l] * W[l], 256), 256, 0, st>>>(L, l, k1, v1);
                ORP_LAUNCHED();
            }
        ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb1, k1, k2, v1, v2, (int)nsort, 0, 64, st));
        count_launches(9);
    }
    const int dgrid = (int)ceil_div((long long)B * S, 128);
    if (aug) decode_kernel<true><<<dgrid, 128, 0, st>>>(L, v2, score_thr, nullptr, view_meta, O);
    else decode_kernel<false><<<dgrid, 128, 0, st>>>(L, v2, score_thr, scale_factor, nullptr, O);
    ORP_LAUNCHED();
    int32_t *nms_ovf = Sc.get<int32_t>(1);
    if (!nms_ovf) return fail(ORP_ECUDA, "%s: scratch allocation failed", who);
    ORP_CUDA(cudaMemsetAsync(nms_ovf, 0, sizeof(int32_t), st));
    rc = run_nms(O.dets, O.segs, (int)total, iou_thr, ORP_NMS_EXACT64, ORP_UNION_NAN_KEEPS, ORP_ORDER_INDEX_ASC, nullptr,
                 nullptr, st, keep, true, B * num_cls, nms_ovf);
    if (rc) return rc;
    ORP_CUDA(cudaMemsetAsync(counts, 0, sizeof(int32_t) * B, st));
    count_kernel<<<dim3(32, B), 256, 0, st>>>(keep, O.valid, (int)per_img, B, counts);
    ORP_LAUNCHED();
    select_keys_kernel<<<grid_for(total, 256), 256, 0, st>>>(keep, O.valid, O.dets, counts, (int)per_img, B, max_per_img, sk1, sv1);
    ORP_LAUNCHED();
    ORP_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb2, sk1, sk2, sv1, sv2, (int)total, 0, sel_bits, st));
    count_launches((sel_bits + 7) / 8 + 1);
    gather_kernel<<<dim3(ceil_div(max_per_img, 128), B), 128, 0, st>>>(sv2, counts, O.dets, O.rp, O.box, out_scale, (int)per_img,
                                                                     (int)S, num_cls, max_per_img, B, dets_out, labels_out,
                                                                     counts_out, nms_ovf);
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace
}  // namespace orp

extern "C" int orp_head_postprocess(int nlevels, const float *const *cls, const float *const *ref, const int *H,
                                    const int *W, const int *stride, int B, int num_cls, int nms_pre, float score_thr,
                                    double iou_thr, int max_per_img, const float *scale_factor, float *dets_out,
                                    int64_t *labels_out, int32_t *counts_out, void *stream)
{
    return head_post("orp_head_postprocess", 1, nlevels, cls, ref, H, W, stride, B, num_cls, nms_pre, score_thr, iou_thr,
                     max_per_img, scale_factor, nullptr, nullptr, dets_out, labels_out, counts_out, stream);
}

extern "C" int orp_head_postprocess_aug(int nviews, int nlevels, const float *const *cls, const float *const *ref,
                                        const int *H, const int *W, const int *stride, int B, int num_cls, int nms_pre,
                                        float score_thr, double iou_thr, int max_per_img, const float *view_meta,
                                        const float *out_scale, float *dets_out, int64_t *labels_out, int32_t *counts_out,
                                        void *stream)
{
    if (!view_meta) return fail(ORP_EINVAL, "orp_head_postprocess_aug: view_meta is NULL");
    return head_post("orp_head_postprocess_aug", nviews, nlevels, cls, ref, H, W, stride, B, num_cls, nms_pre, score_thr,
                     iou_thr, max_per_img, nullptr, view_meta, out_scale, dets_out, labels_out, counts_out, stream);
}

extern "C" int orp_pack_detections(const float *dets, const int64_t *labels, const int32_t *counts, int B, int max_per_img,
                                   float *packed_out, void *stream)
{
    if (!dets || !labels || !counts || !packed_out || B < 1 || max_per_img < 1) return fail(ORP_EINVAL, "orp_pack_detections: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const size_t total = (size_t)B * (max_per_img + 1) * 28;
    pack_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(dets, labels, counts, B, max_per_img, packed_out);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_dcn_offsets_multi(int nprob, const float *const *pts, float *const *off, const long long *numel,
                                     float gradient_mul, const float *base18, void *stream)
{
    if (nprob < 1 || nprob > 8 || !pts || !off || !numel || !base18) return fail(ORP_EINVAL, "orp_dcn_offsets_multi: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    OffsetParams P;
    memset(&P, 0, sizeof(P));
    P.nprob = nprob; P.g = gradient_mul;
    long long mx = 0;
    for (int i = 0; i < nprob; ++i) {
        if (!pts[i] || !off[i] || numel[i] < 0 || numel[i] % 18) return fail(ORP_EINVAL, "orp_dcn_offsets_multi: bad problem");
        P.p[i].pts = pts[i]; P.p[i].off = off[i]; P.p[i].n = numel[i];
        mx = numel[i] > mx ? numel[i] : mx;
    }
    for (int c = 0; c < 18; ++c) P.base[c] = base18[c];
    if (mx == 0) return ORP_OK;
    dim3 grid((unsigned)grid_for((size_t)mx, 256), (unsigned)nprob);
    dcn_offsets_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}
