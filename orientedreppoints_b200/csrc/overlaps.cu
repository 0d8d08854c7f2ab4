// overlaps.cu - pairwise rotated IoU matrices for sm_90a (SURVEY.md section 8 rows a13, a15, n2).
//
//   orp_poly_overlaps(_host)   DOTA_devkit/poly_nms_gpu/poly_overlaps_kernel.cu:280-427
//   orp_quad_iou_matrix        N x K over 8-coordinate quads (rnms/poly_nms IoU as a matrix)
//   orp_iou_poly_f64_pairs     DOTA_devkit/polyiou.cpp:108-128, batched on the device
//   orp_box_iou_rotated        mmdet/ops/box_iou_rotated/src/box_iou_rotated_cuda.cu:13-62
//
// Layout: row boxes are converted to corners once and staged in shared memory per tile; a block
// computes 32 x 32 output tiles (one column tile, row tiles gridDim.y apart), threadIdx.x runs along K so the fp32 stores are coalesced
// (128 B per warp).  The kernels are bound by the output write (4 B per pair) once the AABB
// early-out removes the clipping work for disjoint pairs.
#include "common.cuh"
#include "geom.cuh"

namespace orp {

// RotBox2Poly (poly_overlaps_kernel.cu:280-297): mixed float/double exactly as the reference
// types it (w / 2.0 is double).  cos/sin of the fp32 angle are evaluated in double and rounded
// to fp32 (the reference calls the fp32 routines; <= 1 ulp apart, see DESIGN.md).
__device__ __forceinline__ void rotbox_to_quad(const float *b, float *q)
{
    const float cs = (float)cos((double)b[4]);
    const float ss = (float)sin((double)b[4]);
    const float w = b[2], h = b[3], xc = b[0], yc = b[1];
    const double hw = w / 2.0, hh = h / 2.0, nhw = -w / 2.0, nhh = -h / 2.0;
    q[0] = (float)__dsub_rn(__dadd_rn((double)xc, __dmul_rn((double)cs, hw)), __dmul_rn((double)ss, nhh));
    q[2] = (float)__dsub_rn(__dadd_rn((double)xc, __dmul_rn((double)cs, hw)), __dmul_rn((double)ss, hh));
    q[4] = (float)__dsub_rn(__dadd_rn((double)xc, __dmul_rn((double)cs, nhw)), __dmul_rn((double)ss, hh));
    q[6] = (float)__dsub_rn(__dadd_rn((double)xc, __dmul_rn((double)cs, nhw)), __dmul_rn((double)ss, nhh));
    q[1] = (float)__dadd_rn(__dadd_rn((double)yc, __dmul_rn((double)ss, hw)), __dmul_rn((double)cs, nhh));
    q[3] = (float)__dadd_rn(__dadd_rn((double)yc, __dmul_rn((double)ss, hw)), __dmul_rn((double)cs, hh));
    q[5] = (float)__dadd_rn(__dadd_rn((double)yc, __dmul_rn((double)ss, nhw)), __dmul_rn((double)cs, hh));
    q[7] = (float)__dadd_rn(__dadd_rn((double)yc, __dmul_rn((double)ss, nhw)), __dmul_rn((double)cs, nhh));
}

__global__ void __launch_bounds__(256)
rotbox_to_quad_kernel(const float *__restrict__ boxes5, int n, float *__restrict__ quads8)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float b[5], q[8];
#pragma unroll
    for (int k = 0; k < 5; ++k) b[k] = boxes5[(size_t)i * 5 + k];
    rotbox_to_quad(b, q);
#pragma unroll
    for (int k = 0; k < 8; ++k) quads8[(size_t)i * 8 + k] = q[k];
}

// IoU value of one quad pair.
//   EXACT64 : fp32 clip in pair-local coordinates; value recomputed by the fp64 reference
//             algorithm when the clip's own error bound exceeds 2e-6 of the union (keeps every
//             value within 1e-5 of polyiou.cpp).
//   COMPAT32: the reference's fp32 arithmetic, bit for bit.
__device__ __forceinline__ float quad_iou_value(const float *a, const float *b, int iou_mode, int union_mode)
{
    if (iou_mode == ORP_NMS_COMPAT32) {
        PairRes<float> r = ref_quad_pair<float>(a, b);
        return iou_from<float>(r, union_mode);
    }
    float axmin = fminf(fminf(a[0], a[2]), fminf(a[4], a[6])), axmax = fmaxf(fmaxf(a[0], a[2]), fmaxf(a[4], a[6]));
    float aymin = fminf(fminf(a[1], a[3]), fminf(a[5], a[7])), aymax = fmaxf(fmaxf(a[1], a[3]), fmaxf(a[5], a[7]));
    float bxmin = fminf(fminf(b[0], b[2]), fminf(b[4], b[6])), bxmax = fmaxf(fmaxf(b[0], b[2]), fmaxf(b[4], b[6]));
    float bymin = fminf(fminf(b[1], b[3]), fminf(b[5], b[7])), bymax = fmaxf(fmaxf(b[1], b[3]), fmaxf(b[5], b[7]));
    const bool overlap = (axmin < bxmax) && (bxmin < axmax) && (aymin < bymax) && (bymin < aymax);
    const float ox = 0.5f * (fmaxf(axmin, bxmin) + fminf(axmax, bxmax));
    const float oy = 0.5f * (fmaxf(aymin, bymin) + fminf(aymax, bymax));
    float la[8], lb[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        la[2 * k] = a[2 * k] - ox; la[2 * k + 1] = a[2 * k + 1] - oy;
        lb[2 * k] = b[2 * k] - ox; lb[2 * k + 1] = b[2 * k + 1] - oy;
    }
    if (!(quad_is_convex(a) && quad_is_convex(b))) {
        // concave / self-intersecting / degenerate: only the reference algorithm defines the answer
    } else if (!overlap) {
        // disjoint hulls: intersection is exactly empty; only the degenerate-union conventions matter
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int j = (i + 1) & 3;
            sa += a[2 * i] * a[2 * j + 1] - a[2 * i + 1] * a[2 * j];
            sb += b[2 * i] * b[2 * j + 1] - b[2 * i + 1] * b[2 * j];
        }
        if (sa != 0.f || sb != 0.f) return 0.f;
    } else {
        FastRes r = fast_quad_pair(la, lb);
        const float uni = r.area_a + r.area_b - r.inter;
        if (uni > 0.f && 3.f * r.err < 2e-6f * uni) return r.inter / uni;
    }
    double p[8], q[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { p[k] = (double)a[k]; q[k] = (double)b[k]; }
    PairRes<double> r = ref_quad_pair<double>(p, q);
    return (float)iou_from<double>(r, union_mode);
}

constexpr int kTile = 32;
// Row tiles sit on grid.y, which stops at 65 535 blocks: a block walks the row tiles gridDim.y apart, so any n
// (N proposals against a few queries is the common use) fits in one launch.
constexpr int kMaxRowBlocks = 65535;

static dim3 pair_grid(int n, int k) { return dim3(ceil_div(k, kTile), ceil_div(n, kTile) < kMaxRowBlocks ? ceil_div(n, kTile) : kMaxRowBlocks); }

__global__ void __launch_bounds__(kTile * 8)
quad_iou_matrix_kernel(const float *__restrict__ qa, int n, const float *__restrict__ qb, int k,
                       int iou_mode, int union_mode, float *__restrict__ out)
{
    __shared__ float sa[kTile][9];
    __shared__ float sb[kTile][9];
    const int c0 = blockIdx.x * kTile;
    const int tid = threadIdx.y * kTile + threadIdx.x;   // 256 threads
    const int srow = tid >> 3, sc = tid & 7;
    if (c0 + srow < k) sb[srow][sc] = qb[(size_t)(c0 + srow) * 8 + sc];
    const int col = c0 + threadIdx.x;
    for (long long r0 = (long long)blockIdx.y * kTile; r0 < n; r0 += (long long)gridDim.y * kTile) {
        if (r0 + srow < n) sa[srow][sc] = qa[(size_t)(r0 + srow) * 8 + sc];
        __syncthreads();
        if (col < k) {
            float b[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) b[c] = sb[threadIdx.x][c];
#pragma unroll 1
            for (int rr = threadIdx.y; rr < kTile; rr += 8) {
                const long long row = r0 + rr;
                if (row >= n) break;
                float a[8];
#pragma unroll
                for (int c = 0; c < 8; ++c) a[c] = sa[rr][c];
                out[(size_t)row * k + col] = quad_iou_value(a, b, iou_mode, union_mode);
            }
        }
        __syncthreads();                                  // the tile's rows are consumed before the next one is staged
    }
}

__global__ void __launch_bounds__(128)
iou_poly_f64_pairs_kernel(const double *__restrict__ p, const double *__restrict__ q, int n,
                          double *__restrict__ out)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double a[8], b[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { a[k] = p[(size_t)i * 8 + k]; b[k] = q[(size_t)i * 8 + k]; }
    PairRes<double> r = ref_quad_pair<double>(a, b);
    out[i] = iou_from<double>(r, ORP_UNION_NAN_KEEPS);
}

// detectron2-style boxes: vertices as get_rotated_vertices (box_iou_rotated_utils.h:55-75) after the
// centre shift of single_box_iou_rotated (:317-330); areas are w*h (:332-336).
__global__ void __launch_bounds__(kTile * 8)
box_iou_rotated_kernel(const float *__restrict__ b1, int n, const float *__restrict__ b2, int m,
                       float *__restrict__ out)
{
    __shared__ float s1[kTile][5];
    __shared__ float s2[kTile][5];
    const int c0 = blockIdx.x * kTile;
    const int tid = threadIdx.y * kTile + threadIdx.x;
    const int srow = tid / 5, sc = tid % 5;
    if (tid < kTile * 5 && c0 + srow < m) s2[srow][sc] = b2[(size_t)(c0 + srow) * 5 + sc];
    const int col = c0 + threadIdx.x;
    for (long long r0 = (long long)blockIdx.y * kTile; r0 < n; r0 += (long long)gridDim.y * kTile) {
        if (tid < kTile * 5 && r0 + srow < n) s1[srow][sc] = b1[(size_t)(r0 + srow) * 5 + sc];
        __syncthreads();
        if (col < m) {
            const float x2 = s2[threadIdx.x][0], y2 = s2[threadIdx.x][1], w2 = s2[threadIdx.x][2], h2 = s2[threadIdx.x][3];
            float sn2, cs2;
            sincosf(s2[threadIdx.x][4], &sn2, &cs2);
#pragma unroll 1
            for (int rr = threadIdx.y; rr < kTile; rr += 8) {
                const long long row = r0 + rr;
                if (row >= n) break;
                const float x1 = s1[rr][0], y1 = s1[rr][1], w1 = s1[rr][2], h1 = s1[rr][3];
                const float area1 = w1 * h1, area2 = w2 * h2;
                float res = 0.f;
                // the float areas against the double literal, as box_iou_rotated_utils.h:334 compares them: an area of
                // exactly (float)1e-14 is below 1e-14 and gives 0
                if (!((double)area1 < 1e-14 || (double)area2 < 1e-14)) {
                    float sn1, cs1;
                    sincosf(s1[rr][4], &sn1, &cs1);
                    const float sx = 0.5f * (x1 + x2), sy = 0.5f * (y1 + y2);
                    float a[8], b[8];
                    {
                        const float xc = x1 - sx, yc = y1 - sy, c = 0.5f * cs1, s = 0.5f * sn1;
                        a[0] = xc - s * h1 - c * w1; a[1] = yc + c * h1 - s * w1;
                        a[2] = xc + s * h1 - c * w1; a[3] = yc - c * h1 - s * w1;
                        a[4] = 2.f * xc - a[0]; a[5] = 2.f * yc - a[1];
                        a[6] = 2.f * xc - a[2]; a[7] = 2.f * yc - a[3];
                    }
                    {
                        const float xc = x2 - sx, yc = y2 - sy, c = 0.5f * cs2, s = 0.5f * sn2;
                        b[0] = xc - s * h2 - c * w2; b[1] = yc + c * h2 - s * w2;
                        b[2] = xc + s * h2 - c * w2; b[3] = yc - c * h2 - s * w2;
                        b[4] = 2.f * xc - b[0]; b[5] = 2.f * yc - b[1];
                        b[6] = 2.f * xc - b[2]; b[7] = 2.f * yc - b[3];
                    }
                    // disjoint corner hulls: the intersection is empty.  The clip alone does not give 0 when the centre
                    // shift has collapsed a tiny box onto one fp32 point far from the other (the reference returns
                    // garbage there, up to inf)
                    const float axmin = fminf(fminf(a[0], a[2]), fminf(a[4], a[6])), axmax = fmaxf(fmaxf(a[0], a[2]), fmaxf(a[4], a[6]));
                    const float aymin = fminf(fminf(a[1], a[3]), fminf(a[5], a[7])), aymax = fmaxf(fmaxf(a[1], a[3]), fmaxf(a[5], a[7]));
                    const float bxmin = fminf(fminf(b[0], b[2]), fminf(b[4], b[6])), bxmax = fmaxf(fmaxf(b[0], b[2]), fmaxf(b[4], b[6]));
                    const float bymin = fminf(fminf(b[1], b[3]), fminf(b[5], b[7])), bymax = fmaxf(fmaxf(b[1], b[3]), fmaxf(b[5], b[7]));
                    if (axmin < bxmax && bxmin < axmax && aymin < bymax && bymin < aymax) {
                        FastRes r = fast_quad_pair(a, b);
                        res = r.inter / (area1 + area2 - r.inter);
                    }
                }
                out[(size_t)row * m + col] = res;
            }
        }
        __syncthreads();                                  // the tile's rows are consumed before the next one is staged
    }
}

static int quad_matrix(const float *qa, int n, const float *qb, int k, int iou_mode, int union_mode,
                       float *out, cudaStream_t st)
{
    if (n == 0 || k == 0) return ORP_OK;
    quad_iou_matrix_kernel<<<pair_grid(n, k), dim3(kTile, 8), 0, st>>>(qa, n, qb, k, iou_mode, union_mode, out);
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace orp

using namespace orp;

extern "C" int orp_quad_iou_matrix(const float *quads_a, int n, const float *quads_b, int k, int iou_mode,
                                   int union_mode, float *out, void *stream)
{
    if (n < 0 || k < 0 || ((n > 0 && k > 0) && (!quads_a || !quads_b || !out)))
        return fail(ORP_EINVAL, "orp_quad_iou_matrix: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    return quad_matrix(quads_a, n, quads_b, k, iou_mode, union_mode, out, static_cast<cudaStream_t>(stream));
}

extern "C" int orp_poly_overlaps(const float *boxes5, int n, const float *query5, int k, float *out, void *stream)
{
    if (n < 0 || k < 0 || ((n > 0 && k > 0) && (!boxes5 || !query5 || !out)))
        return fail(ORP_EINVAL, "orp_poly_overlaps: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    if (n == 0 || k == 0) return ORP_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    Scratch S(st);
    float *qa = S.get<float>((size_t)n * 8), *qb = S.get<float>((size_t)k * 8);
    if (!qa || !qb) return fail(ORP_ECUDA, "orp_poly_overlaps: scratch allocation failed");
    rotbox_to_quad_kernel<<<ceil_div(n, 256), 256, 0, st>>>(boxes5, n, qa);
    ORP_LAUNCHED();
    rotbox_to_quad_kernel<<<ceil_div(k, 256), 256, 0, st>>>(query5, k, qb);
    ORP_LAUNCHED();
    return quad_matrix(qa, n, qb, k, ORP_NMS_EXACT64, ORP_UNION_GUARD, out, st);
}

extern "C" int orp_poly_overlaps_host(float *overlaps, const float *boxes, const float *query_boxes, int n,
                                      int k, int device_id)
{
    if (n < 0 || k < 0 || ((n > 0 && k > 0) && (!overlaps || !boxes || !query_boxes)))
        return fail(ORP_EINVAL, "orp_poly_overlaps_host: bad arguments");
    if (n == 0 || k == 0) return ORP_OK;
    int prev = 0;
    ORP_CUDA(cudaGetDevice(&prev));
    ORP_CUDA(cudaSetDevice(device_id));
    cudaStream_t st;
    ORP_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    float *db = nullptr, *dq = nullptr, *dout = nullptr;
    int rc = ORP_OK;
    do {
        if (cudaMallocAsync(&db, sizeof(float) * 5 * (size_t)n, st) != cudaSuccess ||
            cudaMallocAsync(&dq, sizeof(float) * 5 * (size_t)k, st) != cudaSuccess ||
            cudaMallocAsync(&dout, sizeof(float) * (size_t)n * k, st) != cudaSuccess) { rc = fail(ORP_ECUDA, "orp_poly_overlaps_host: alloc"); break; }
        cudaMemcpyAsync(db, boxes, sizeof(float) * 5 * (size_t)n, cudaMemcpyHostToDevice, st);
        cudaMemcpyAsync(dq, query_boxes, sizeof(float) * 5 * (size_t)k, cudaMemcpyHostToDevice, st);
        rc = orp_poly_overlaps(db, n, dq, k, dout, st);
        if (rc) break;
        if (cudaMemcpyAsync(overlaps, dout, sizeof(float) * (size_t)n * k, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess) { rc = fail(ORP_ECUDA, "orp_poly_overlaps_host: d2h"); break; }
    } while (0);
    if (db) cudaFreeAsync(db, st);
    if (dq) cudaFreeAsync(dq, st);
    if (dout) cudaFreeAsync(dout, st);
    cudaStreamSynchronize(st);
    cudaStreamDestroy(st);
    cudaSetDevice(prev);
    return rc;
}

extern "C" int orp_iou_poly_f64_pairs(const double *p8, const double *q8, int n, double *out, void *stream)
{
    if (n < 0 || (n > 0 && (!p8 || !q8 || !out))) return fail(ORP_EINVAL, "orp_iou_poly_f64_pairs: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    if (n == 0) return ORP_OK;
    iou_poly_f64_pairs_kernel<<<ceil_div(n, 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(p8, q8, n, out);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_box_iou_rotated(const float *boxes1, int n, const float *boxes2, int m, float *out, void *stream)
{
    if (n < 0 || m < 0 || ((n > 0 && m > 0) && (!boxes1 || !boxes2 || !out)))
        return fail(ORP_EINVAL, "orp_box_iou_rotated: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    if (n == 0 || m == 0) return ORP_OK;
    box_iou_rotated_kernel<<<pair_grid(n, m), dim3(kTile, 8), 0, static_cast<cudaStream_t>(stream)>>>(boxes1, n, boxes2, m, out);
    ORP_LAUNCHED();
    return ORP_OK;
}
