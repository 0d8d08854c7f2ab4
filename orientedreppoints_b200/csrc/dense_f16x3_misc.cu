// dense_f16x3_misc.cu - the memory-bound companions of the f16x3 ("split") tensor-core convolutions.
//
// A split tensor carries every fp32 value as an fp16 pair x = hi + lo, laid out [N,H,W,2,C]: per pixel the C hi
// values, then the C lo values (the stem's space-to-depth input is plane-separated instead: [2][N,H',W',16]).
// Everything here reads pairs, computes in fp32 exactly as the reference's fp32 layers do (max-pool
// resnet.py:497, GroupNorm ops/norm.py:42-50 + FPN top-down add fpn.py:171-176, Normalize of the test pipeline)
// and writes pairs.  All HBM-bound: 16-byte vector accesses, grids sized in multiples of the SM count.
#include <cuda_fp16.h>
#include <cstring>

#include "common.cuh"

namespace orp {
namespace {

// 8 values <- 16 bytes of hi + 16 bytes of lo
__device__ __forceinline__ void join8(const uint4 &h, const uint4 &l, float (&o)[8])
{
    const uint32_t hh[4] = {h.x, h.y, h.z, h.w}, ll[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&hh[k]));
        const float2 b = __half22float2(*reinterpret_cast<const __half2 *>(&ll[k]));
        o[2 * k] = a.x + b.x;                 // exact: the pair has at most 22 significant bits
        o[2 * k + 1] = a.y + b.y;
    }
}
// 8 values -> (hi, lo); values beyond the fp16 range saturate (the convolutions count such events)
__device__ __forceinline__ void split8(const float (&v)[8], uint4 &h, uint4 &l)
{
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float a = fminf(fmaxf(v[2 * k], -65504.f), 65504.f), b = fminf(fmaxf(v[2 * k + 1], -65504.f), 65504.f);
        const __half2 h2 = __floats2half2_rn(a, b);
        const float2 hf = __half22float2(h2);
        const __half2 l2 = __floats2half2_rn(a - hf.x, b - hf.y);
        hh[k] = *reinterpret_cast<const uint32_t *>(&h2);
        ll[k] = *reinterpret_cast<const uint32_t *>(&l2);
    }
    h = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    l = make_uint4(ll[0], ll[1], ll[2], ll[3]);
}

int grid_for(size_t items, int threads)
{
    size_t g = (items + threads - 1) / threads;
    const size_t cap = kNumSMs * 16;
    return (int)(g < cap ? (g ? g : 1) : cap);
}

// fp32 [pixels, C] -> split [pixels, 2, C]
__global__ void __launch_bounds__(256)
split_from_f32_kernel(const float *__restrict__ x, size_t pixels, int C, __half *__restrict__ y)
{
    const int c8 = C / 8;
    const size_t total = pixels * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / c8;
        const int c = (int)(i - pix * c8) * 8;
        const float4 a = *reinterpret_cast<const float4 *>(x + pix * C + c), b = *reinterpret_cast<const float4 *>(x + pix * C + c + 4);
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        uint4 h, l;
        split8(v, h, l);
        *reinterpret_cast<uint4 *>(y + pix * 2 * C + c) = h;
        *reinterpret_cast<uint4 *>(y + pix * 2 * C + C + c) = l;
    }
}

__global__ void __launch_bounds__(256)
split_to_f32_kernel(const __half *__restrict__ x, size_t pixels, int C, float *__restrict__ y)
{
    const int c8 = C / 8;
    const size_t total = pixels * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / c8;
        const int c = (int)(i - pix * c8) * 8;
        float v[8];
        join8(*reinterpret_cast<const uint4 *>(x + pix * 2 * C + c), *reinterpret_cast<const uint4 *>(x + pix * 2 * C + C + c), v);
        *reinterpret_cast<float4 *>(y + pix * C + c) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4 *>(y + pix * C + c + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
}

__global__ void __launch_bounds__(256)
maxpool3x3s2_split_kernel(const __half *__restrict__ x, int N, int H, int W, int C, int Ho, int Wo, __half *__restrict__ y)
{
    const int c8 = C / 8;
    const size_t total = (size_t)N * Ho * Wo * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c8) * 8;
        const size_t pix = i / c8;
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), n = (int)(pix / ((size_t)Wo * Ho));
        float m[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
#pragma unroll
        for (int dh = 0; dh < 3; ++dh)
#pragma unroll
            for (int dw = 0; dw < 3; ++dw) {
                const int ih = oh * 2 - 1 + dh, iw = ow * 2 - 1 + dw;
                if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
                const __half *p = x + (((size_t)n * H + ih) * W + iw) * 2 * C + c;
                float v[8];
                join8(*reinterpret_cast<const uint4 *>(p), *reinterpret_cast<const uint4 *>(p + C), v);
#pragma unroll
                for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
            }
        uint4 h, l;
        split8(m, h, l);                      // the maximum is one of the inputs: re-splitting it is exact
        *reinterpret_cast<uint4 *>(y + pix * 2 * C + c) = h;
        *reinterpret_cast<uint4 *>(y + pix * 2 * C + C + c) = l;
    }
}

// GroupNorm statistics of a split tensor with C = 256, 32 groups (fallback when the convolution epilogue could not fuse them)
__global__ void __launch_bounds__(256)
gn_stats_split_kernel(const __half *__restrict__ x, int HW, int slab, double *__restrict__ stats)
{
    __shared__ float s_sum[8][32], s_sq[8][32];
    const int n = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int p0 = blockIdx.x * slab, p1 = min(HW, p0 + slab);
    const __half *base = x + (size_t)n * HW * 512 + lane * 8;
    float s = 0.f, q = 0.f;
    for (int p = p0 + warp; p < p1; p += 8) {
        float v[8];
        join8(*reinterpret_cast<const uint4 *>(base + (size_t)p * 512), *reinterpret_cast<const uint4 *>(base + (size_t)p * 512 + 256), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) { s += v[j]; q = fmaf(v[j], v[j], q); }
    }
    s_sum[warp][lane] = s;
    s_sq[warp][lane] = q;
    __syncthreads();
    if (warp == 0) {
        double ds = 0, dq = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) { ds += (double)s_sum[w][lane]; dq += (double)s_sq[w][lane]; }
        atomicAdd(&stats[((size_t)n * 32 + lane) * 2], ds);
        atomicAdd(&stats[((size_t)n * 32 + lane) * 2 + 1], dq);
    }
}

struct GnApplyProb {
    const __half *x;
    const double *stats;
    const __half *up;
    __half *y;
    int N, H, W;
    int img_start;                  // first blockIdx.y of this problem
};
struct GnApplyParams {
    GnApplyProb p[8];
    int nprob;
    const float *gamma, *beta;
    float eps;
    int relu;
};

// One (problem, image) per blockIdx.y; item = (pixel, 8-channel group): thread's group = index & 31, so mean / rstd /
// gamma / beta stay in registers.  Per item: 2 x 16 B in, fp32 normalise (+ nearest-neighbour top-down add), 2 x 16 B out.
__global__ void __launch_bounds__(256)
gn_apply_split_kernel(const __grid_constant__ GnApplyParams P)
{
    int pi = 0;
#pragma unroll
    for (int k = 1; k < 8; ++k)
        if (k < P.nprob && (int)blockIdx.y >= P.p[k].img_start) pi = k;
    const GnApplyProb &pr = P.p[pi];
    const int n = (int)blockIdx.y - pr.img_start;
    const int H = pr.H, W = pr.W;
    const uint32_t items = (uint32_t)H * W * 32;
    const uint32_t first = blockIdx.x * 1024u + threadIdx.x;
    if (first >= items) return;
    const int g = threadIdx.x & 31;
    const double cnt = (double)H * W * 8;
    const double sm = pr.stats[((size_t)n * 32 + g) * 2], sq = pr.stats[((size_t)n * 32 + g) * 2 + 1];
    const double mean = sm / cnt;
    double var = sq / cnt - mean * mean;
    var = var < 0 ? 0 : var;
    const float rstd = (float)(1.0 / sqrt(var + (double)P.eps)), mu = (float)mean;
    const float4 g0 = *reinterpret_cast<const float4 *>(P.gamma + g * 8), g1 = *reinterpret_cast<const float4 *>(P.gamma + g * 8 + 4);
    const float4 b0 = *reinterpret_cast<const float4 *>(P.beta + g * 8), b1 = *reinterpret_cast<const float4 *>(P.beta + g * 8 + 4);
    const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    const float be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    const __half *xi = pr.x + (size_t)n * H * W * 512 + g * 8;
    __half *yi = pr.y + (size_t)n * H * W * 512 + g * 8;
    const int Hu = (H + 1) / 2, Wu = (W + 1) / 2;           // F.interpolate(size=prev_shape, mode='nearest'): src = floor(dst * in / out)
    const __half *upi = pr.up ? pr.up + (size_t)n * Hu * Wu * 512 + g * 8 : nullptr;
    uint4 uh[4], ul[4];
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const uint32_t i = first + it * 256u;
        if (i < items) {
            const size_t hw = i >> 5;
            uh[it] = *reinterpret_cast<const uint4 *>(xi + hw * 512);
            ul[it] = *reinterpret_cast<const uint4 *>(xi + hw * 512 + 256);
        }
    }
#pragma unroll
    for (int it = 0; it < 4; ++it) {
        const uint32_t i = first + it * 256u;
        if (i >= items) break;
        const size_t hw = i >> 5;
        float o[8];
        join8(uh[it], ul[it], o);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[j] = (o[j] - mu) * rstd * ga[j] + be[j];
            if (P.relu) o[j] = fmaxf(o[j], 0.f);
        }
        if (upi) {
            const int h = (int)(hw / W), w = (int)(hw - (size_t)h * W);
            const __half *up = upi + ((size_t)((h * Hu) / H) * Wu + (w * Wu) / W) * 512;
            float t[8];
            join8(*reinterpret_cast<const uint4 *>(up), *reinterpret_cast<const uint4 *>(up + 256), t);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += t[j];
        }
        uint4 h4, l4;
        split8(o, h4, l4);
        *reinterpret_cast<uint4 *>(yi + hw * 512) = h4;
        *reinterpret_cast<uint4 *>(yi + hw * 512 + 256) = l4;
    }
}

// Space-to-depth form of the stem input as two fp16 planes [2][N,Hp,Wp,16]:
// v[n][Y][X][(dy*2+dx)*3 + c] = img[n][c][2(Y-2)+dy][2(X-2)+dx] (zero outside the image, channels 12-15 zero).
// SRC_U8: decoded uint8 HWC tiles with the test pipeline's Normalize fused (mmcv.imnormalize: optional BGR->RGB,
// (x - mean) * (1/std) in fp32; mean / stdinv indexed by MODEL channel).  valid (SRC_U8 only; int32 [N,2] = (h, w) per
// image, or null for the full extent): pixels at y >= h or x >= w are the pipeline's Pad after Normalize, exactly 0.0.
template <bool SRC_U8>
__global__ void __launch_bounds__(256)
stem_s2d_split_kernel(const void *__restrict__ img_v, int N, int H, int W, float3 mean, float3 stdinv, int to_rgb,
                      const int32_t *__restrict__ valid, __half *__restrict__ out)
{
    const int Hp = H / 2 + 3, Wp = W / 2 + 3;
    const size_t total = (size_t)N * Hp * Wp;
    const float mu[3] = {mean.x, mean.y, mean.z}, si[3] = {stdinv.x, stdinv.y, stdinv.z};
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int X = (int)(i % Wp);
        const size_t t = i / Wp;
        const int Y = (int)(t % Hp), n = (int)(t / Hp);
        const int y0 = 2 * (Y - 2), x0 = 2 * (X - 2);
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = 0.f;
        const int vh = valid ? min(valid[2 * n], H) : H, vw = valid ? min(valid[2 * n + 1], W) : W;
        if (x0 >= 0 && x0 < vw) {                                             // W is even: x0 + 1 < W
#pragma unroll
            for (int dy = 0; dy < 2; ++dy) {
                const int y = y0 + dy;
                if (y < 0 || y >= vh) continue;
                if (SRC_U8) {
                    const uint8_t *p = static_cast<const uint8_t *>(img_v) + (((size_t)n * H + y) * W + x0) * 3;   // 6 bytes, even address
                    const uint16_t a = *reinterpret_cast<const uint16_t *>(p), b = *reinterpret_cast<const uint16_t *>(p + 2),
                                   c2 = *reinterpret_cast<const uint16_t *>(p + 4);
                    const uint8_t px[6] = {(uint8_t)(a & 0xff), (uint8_t)(a >> 8), (uint8_t)(b & 0xff), (uint8_t)(b >> 8),
                                           (uint8_t)(c2 & 0xff), (uint8_t)(c2 >> 8)};
#pragma unroll
                    for (int dx = 0; dx < 2; ++dx) {
                        if (x0 + dx >= vw) continue;                          // odd valid width: the second pixel is padding
#pragma unroll
                        for (int c = 0; c < 3; ++c) {
                            const int sc = to_rgb ? 2 - c : c;
                            v[(dy * 2 + dx) * 3 + c] = ((float)px[dx * 3 + sc] - mu[c]) * si[c];
                        }
                    }
                } else {
                    const float *img = static_cast<const float *>(img_v);
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float2 p = *reinterpret_cast<const float2 *>(img + (((size_t)n * 3 + c) * H + y) * W + x0);
                        v[(dy * 2 + 0) * 3 + c] = p.x;
                        v[(dy * 2 + 1) * 3 + c] = p.y;
                    }
                }
            }
        }
        const float v0[8] = {v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7]};
        const float v1[8] = {v[8], v[9], v[10], v[11], v[12], v[13], v[14], v[15]};
        uint4 h0, l0, h1, l1;
        split8(v0, h0, l0);
        split8(v1, h1, l1);
        uint4 *oh = reinterpret_cast<uint4 *>(out + i * 16), *ol = reinterpret_cast<uint4 *>(out + (total + i) * 16);
        oh[0] = h0; oh[1] = h1;
        ol[0] = l0; ol[1] = l1;
    }
}


// ---- layout conversions at the operator boundary (the reference's ops take NCHW fp32, mmdet/ops/dcn/deform_conv.py:17-58)
// per image a [R, Cc] row-major matrix -> its transpose [Cc, R]; 32 x 32 tiles through shared memory, both sides coalesced
// MODE 0: fp32 -> fp32.  MODE 1: fp32 [C, HW] -> split fp16 [HW, 2, C] (rows = channels, columns = pixels)
template <int MODE>
__global__ void __launch_bounds__(256)
transpose_kernel(const float *__restrict__ x, int R, int Cc, void *__restrict__ yv)
{
    __shared__ float t[32][33];
    const int n = blockIdx.z;
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;             // 32 x 8
    const float *xi = x + (size_t)n * R * Cc;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int r = r0 + ty + k * 8, c = c0 + tx;
        t[ty + k * 8][tx] = (r < R && c < Cc) ? xi[(size_t)r * Cc + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = c0 + ty + k * 8, r = r0 + tx;                      // output row = input column
        if (c < Cc && r < R) {
            const float v = t[tx][ty + k * 8];
            if (MODE == 0) {
                static_cast<float *>(yv)[(size_t)n * R * Cc + (size_t)c * R + r] = v;
            } else {
                const float a = fminf(fmaxf(v, -65504.f), 65504.f);
                const __half h = __float2half_rn(a);
                __half *y = static_cast<__half *>(yv) + ((size_t)n * Cc + c) * 2 * R;   // pixel c: [2][R channels]
                y[r] = h;
                y[R + r] = __float2half_rn(a - __half2float(h));
            }
        }
    }
}

}  // namespace
}  // namespace orp

using namespace orp;

extern "C" int orp_split_from_f32(const float *x, long long pixels, int C, void *y_split, void *stream)
{
    if (!x || !y_split || pixels < 0 || C < 8 || C % 8) return fail(ORP_EINVAL, "split_from_f32: C must be a multiple of 8");
    if (pixels == 0) return ORP_OK;
    int rc = ensure_device();
    if (rc) return rc;
    split_from_f32_kernel<<<grid_for((size_t)pixels * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        x, (size_t)pixels, C, static_cast<__half *>(y_split));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_split_to_f32(const void *x_split, long long pixels, int C, float *y, void *stream)
{
    if (!x_split || !y || pixels < 0 || C < 8 || C % 8) return fail(ORP_EINVAL, "split_to_f32: C must be a multiple of 8");
    if (pixels == 0) return ORP_OK;
    int rc = ensure_device();
    if (rc) return rc;
    split_to_f32_kernel<<<grid_for((size_t)pixels * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __half *>(x_split), (size_t)pixels, C, y);
    ORP_LAUNCHED();
    return ORP_OK;
}

static int stem_s2d_u8_f16x3_impl(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std, int to_rgb,
                                  const int32_t *valid, void *out, void *stream)
{
    if (!img_hwc || !out || !mean || !std || N < 1 || H < 2 || W < 2 || (H & 1) || (W & 1))
        return fail(ORP_EINVAL, "stem_s2d_u8_f16x3: needs even H, W");
    int rc = ensure_device();
    if (rc) return rc;
    const float3 mu = make_float3(mean[0], mean[1], mean[2]);
    // mmcv.imnormalize: stdinv = 1 / np.float64(std), applied to the float32 image
    const float3 si = make_float3((float)(1.0 / (double)std[0]), (float)(1.0 / (double)std[1]), (float)(1.0 / (double)std[2]));
    const size_t total = (size_t)N * (H / 2 + 3) * (W / 2 + 3);
    stem_s2d_split_kernel<true><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img_hwc, N, H, W, mu, si, to_rgb, valid, static_cast<__half *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_stem_s2d_u8_f16x3(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                     int to_rgb, void *out, void *stream)
{
    return stem_s2d_u8_f16x3_impl(img_hwc, N, H, W, mean, std, to_rgb, nullptr, out, stream);
}

extern "C" int orp_stem_s2d_u8_padded_f16x3(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                            int to_rgb, const int32_t *valid_hw, void *out, void *stream)
{
    if (!valid_hw) return fail(ORP_EINVAL, "stem_s2d_u8_padded_f16x3: valid_hw is required");
    return stem_s2d_u8_f16x3_impl(img_hwc, N, H, W, mean, std, to_rgb, valid_hw, out, stream);
}

extern "C" int orp_stem_s2d_f16x3(const float *img_nchw, int N, int H, int W, void *out, void *stream)
{
    if (!img_nchw || !out || N < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return fail(ORP_EINVAL, "stem_s2d_f16x3: needs even H, W");
    int rc = ensure_device();
    if (rc) return rc;
    const size_t total = (size_t)N * (H / 2 + 3) * (W / 2 + 3);
    const float3 z = make_float3(0.f, 0.f, 0.f);
    stem_s2d_split_kernel<false><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img_nchw, N, H, W, z, z, 0, nullptr, static_cast<__half *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_maxpool3x3s2_f16x3(const void *x, int N, int H, int W, int C, void *y, void *stream)
{
    if (!x || !y || C % 8) return fail(ORP_EINVAL, "maxpool3x3s2_f16x3: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const size_t total = (size_t)N * Ho * Wo * (C / 8);
    maxpool3x3s2_split_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __half *>(x), N, H, W, C, Ho, Wo, static_cast<__half *>(y));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_stats_f16x3(const void *x, int N, int HW, int C, int groups, double *stats, void *stream)
{
    if (!x || !stats || C != 256 || groups != 32) return fail(ORP_EINVAL, "gn_stats_f16x3: needs C=256, 32 groups");
    int rc = ensure_device();
    if (rc) return rc;
    int slabs = ceil_div(HW, 64);
    const int maxs = (kNumSMs * 4 + N - 1) / N;
    if (slabs > maxs) slabs = maxs;
    const int slab = ceil_div(HW, slabs);
    slabs = ceil_div(HW, slab);
    gn_stats_split_kernel<<<dim3(slabs, N), 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const __half *>(x), HW, slab, stats);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_apply_f16x3_multi(int nprob, const orp_gn_problem *probs, int C, int groups, const float *gamma,
                                        const float *beta, float eps, int relu, void *stream)
{
    if (nprob < 1 || nprob > 8 || !probs || !gamma || !beta || C != 256 || groups != 32)
        return fail(ORP_EINVAL, "gn_apply_f16x3: needs 1..8 problems, C=256, 32 groups");
    int rc = ensure_device();
    if (rc) return rc;
    GnApplyParams P;
    memset(&P, 0, sizeof(P));
    P.nprob = nprob; P.gamma = gamma; P.beta = beta; P.eps = eps; P.relu = relu;
    int imgs = 0;
    size_t max_items = 0;
    for (int i = 0; i < nprob; ++i) {
        const orp_gn_problem &q = probs[i];
        if (!q.x || !q.y || !q.stats || q.N < 1 || q.H < 1 || q.W < 1) return fail(ORP_EINVAL, "gn_apply_f16x3: bad problem");
        if ((size_t)q.H * q.W * 32 > 0xffffffffull) return fail(ORP_EINVAL, "gn_apply_f16x3: image too large");
        P.p[i].x = static_cast<const __half *>(q.x);
        P.p[i].stats = q.stats;
        P.p[i].up = static_cast<const __half *>(q.up_src);
        P.p[i].y = static_cast<__half *>(q.y);
        P.p[i].N = q.N; P.p[i].H = q.H; P.p[i].W = q.W;
        P.p[i].img_start = imgs;
        imgs += q.N;
        const size_t c = (size_t)q.H * q.W * 32;
        max_items = c > max_items ? c : max_items;
    }
    if (imgs > 65535) return fail(ORP_EINVAL, "gn_apply_f16x3: too many images");
    dim3 grid((unsigned)((max_items + 1023) / 1024), (unsigned)imgs);
    gn_apply_split_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_transpose_f32(const float *x, int N, int R, int Cc, float *y, void *stream)
{
    if (!x || !y || N < 1 || R < 1 || Cc < 1 || N > 65535) return fail(ORP_EINVAL, "transpose_f32: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    dim3 grid((unsigned)ceil_div(Cc, 32), (unsigned)ceil_div(R, 32), (unsigned)N);
    if (grid.y > 65535) return fail(ORP_EINVAL, "transpose_f32: too many rows");
    transpose_kernel<0><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, R, Cc, y);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_nchw_f32_to_split(const float *x, int N, int C, int HW, void *y_split, void *stream)
{
    if (!x || !y_split || N < 1 || C < 8 || (C % 8) || HW < 1 || N > 65535) return fail(ORP_EINVAL, "nchw_f32_to_split: C must be a multiple of 8");
    int rc = ensure_device();
    if (rc) return rc;
    dim3 grid((unsigned)ceil_div(HW, 32), (unsigned)ceil_div(C, 32), (unsigned)N);
    transpose_kernel<1><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, C, HW, y_split);
    ORP_LAUNCHED();
    return ORP_OK;
}
