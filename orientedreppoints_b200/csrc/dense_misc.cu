// dense_misc.cu - the memory-bound companions of the tensor-core convolutions, written once for both activation formats
// (act.cuh): bf16 [N,H,W,C] and the f16x3 "split" format fp16 [N,H,W,2,C].  3x3/2 max-pool (resnet.py:497), GroupNorm
// statistics and apply (+ReLU, + the FPN top-down nearest-2x add; ops/norm.py:42-50, fpn.py:171-176) and the stem's
// space-to-depth input (from the NCHW fp32 image, or from uint8 tiles with the test pipeline's Normalize fused).  Only
// the bf16 engine has the stem im2col; only the split format has the fp32 <-> split conversions at the operator boundary.
// Everything computes in fp32 exactly as the reference's fp32 layers do.  All HBM-bound: 16-byte vector accesses, grids
// sized in multiples of the SM count.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstring>

#include "act.cuh"
#include "common.cuh"
#include "../../include/orp_b200_dcnv2.h"

namespace orp {
namespace {

constexpr const char *fmt_name(bool split) { return split ? "f16x3" : "bf16"; }

// img: NCHW fp32 [N,3,H,W] (the layout the reference feeds its backbone) -> bf16 [N,Ho,Wo,192]
// with k = (kh*7 + kw)*3 + c for k < 147 and zeros above: conv1 (resnet.py:495) becomes a 1x1
// convolution over 192 channels on the tensor cores.
// One block = 64 consecutive output pixels of one output row: the 7 x 133 x 3 input patch is staged in shared
// memory with coalesced loads, then every thread emits whole 16-byte chunks (8 k-values) - consecutive threads
// write consecutive chunks of the same 384-byte row, so both sides of the kernel move full cache lines.
constexpr int kStemPix = 64;
__global__ void __launch_bounds__(256)
stem_im2col_kernel(const float *__restrict__ img, int N, int H, int W, int Ho, int Wo, __nv_bfloat16 *__restrict__ out)
{
    constexpr int PW = 2 * kStemPix + 5;                 // 133 input columns
    __shared__ float s_p[3 * 7 * PW];
    __shared__ __align__(16) int s_koff[192];
    const int t = threadIdx.x;
    const int wblocks = (Wo + kStemPix - 1) / kStemPix;
    const int wb = blockIdx.x % wblocks;
    const int oh = (blockIdx.x / wblocks) % Ho, n = blockIdx.x / (wblocks * Ho);
    const int ow0 = wb * kStemPix, x0 = ow0 * 2 - 3, y0 = oh * 2 - 3;
    if (t < 192) {
        const int tap = t / 3, c = t - tap * 3, kh = tap / 7, kw = tap - kh * 7;
        s_koff[t] = t < 147 ? (c * 7 + kh) * PW + kw : -1;
    }
#pragma unroll
    for (int r = 0; r < 21; ++r) {                        // (channel, patch row): warp-uniform decode, coalesced along x
        const int c = r / 7, py = r - c * 7, yy = y0 + py;
        const bool rok = yy >= 0 && yy < H;
        const float *src = img + (((size_t)n * 3 + c) * H + (rok ? yy : 0)) * W;
        if (t < PW) {
            const int xx = x0 + t;
            s_p[r * PW + t] = (rok && xx >= 0 && xx < W) ? __ldg(src + xx) : 0.f;
        }
    }
    __syncthreads();
    const int npix = min(kStemPix, Wo - ow0);
    __nv_bfloat16 *orow = out + (((size_t)n * Ho + oh) * Wo + ow0) * 192;
    for (int item = t; item < npix * 24; item += 256) {
        const int px = item / 24, ck = item - px * 24;
        const int4 o0 = *reinterpret_cast<const int4 *>(&s_koff[ck * 8]), o1 = *reinterpret_cast<const int4 *>(&s_koff[ck * 8 + 4]);
        const int off[8] = {o0.x, o0.y, o0.z, o0.w, o1.x, o1.y, o1.z, o1.w};
        const float *pb = s_p + px * 2;
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = off[j] >= 0 ? pb[off[j]] : 0.f;
        Act<false>::st8(orow + (size_t)item * 8, 0, v);
    }
}

template <bool SPLIT>
__global__ void __launch_bounds__(256)
maxpool3x3s2_kernel(const typename Act<SPLIT>::T *__restrict__ x, int N, int H, int W, int C, int Ho, int Wo,
                    typename Act<SPLIT>::T *__restrict__ y)
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
                float v[8];
                Act<SPLIT>::ld8(x, ((size_t)n * H + ih) * W + iw, C, c, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) m[j] = fmaxf(m[j], v[j]);
            }
        Act<SPLIT>::st8(y, pix, C, c, m);     // the maximum is one of the inputs: re-splitting it is exact
    }
}

// GroupNorm statistics with C = 256, 32 groups (8 channels = one 16-byte vector = one lane): grid (slabs, N); every warp
// strides over the pixels of its slab, lane l owns group l.  (Split format: the fallback when the convolution epilogue
// could not fuse them.)
template <bool SPLIT>
__global__ void __launch_bounds__(256)
gn_stats_kernel(const typename Act<SPLIT>::T *__restrict__ x, int HW, int slab, double *__restrict__ stats)
{
    __shared__ float s_sum[8][32], s_sq[8][32];
    const int n = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int p0 = blockIdx.x * slab, p1 = min(HW, p0 + slab);
    float s = 0.f, q = 0.f;
    for (int p = p0 + warp; p < p1; p += 8) {
        float v[8];
        Act<SPLIT>::ld8(x, (size_t)n * HW + p, 256, lane * 8, v);
        // the two formats keep their own summation order: changing either would change the statistics
        if constexpr (SPLIT) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { s += v[j]; q = fmaf(v[j], v[j], q); }
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                s += v[2 * k] + v[2 * k + 1];
                q += v[2 * k] * v[2 * k] + v[2 * k + 1] * v[2 * k + 1];
            }
        }
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

template <typename T> struct GnApplyProb {
    const T *x;
    const double *stats;
    const T *up;
    T *y;
    int N, H, W;
    int img_start;                  // first blockIdx.y of this problem
};
template <typename T> struct GnApplyParams {
    GnApplyProb<T> p[8];
    int nprob;
    const float *gamma, *beta;
    float eps;
    int relu;
};

// (pixel, 8-channel group) items per thread of the GroupNorm apply: 16 B (bf16) or 32 B (split) each
template <bool SPLIT> constexpr int kGnApplyIt = SPLIT ? 4 : 8;

// One (problem, image) per blockIdx.y.  A thread always works on the same channel group (its index & 31), so the
// group's mean / rstd and the eight gamma / beta values live in registers; per item the work is one load, eight
// multiply-adds, the optional nearest-neighbour top-down add (fpn.py:171-176) and one store.  Three blocks per SM.
template <bool SPLIT>
__global__ void __launch_bounds__(256, 3)
gn_apply_kernel(const __grid_constant__ GnApplyParams<typename Act<SPLIT>::T> P)
{
    constexpr int kIt = kGnApplyIt<SPLIT>;
    int pi = 0;
#pragma unroll
    for (int k = 1; k < 8; ++k)
        if (k < P.nprob && (int)blockIdx.y >= P.p[k].img_start) pi = k;
    const auto &pr = P.p[pi];
    const int n = (int)blockIdx.y - pr.img_start;
    const int H = pr.H, W = pr.W;
    const uint32_t items = (uint32_t)H * W * 32;
    const uint32_t first = blockIdx.x * (kIt * 256u) + threadIdx.x;
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
    const size_t img = (size_t)n * H * W;                      // first pixel of this image
    const int Hu = (H + 1) / 2, Wu = (W + 1) / 2;           // F.interpolate(size=prev_shape, mode='nearest'): src = floor(dst * in / out)
    const size_t up_img = (size_t)n * Hu * Wu;
    // all loads before the first use; items past the image's end re-read its last pixel (in bounds, never stored)
    float v[kIt][8];
#pragma unroll
    for (int it = 0; it < kIt; ++it)
        Act<SPLIT>::ld8(pr.x, img + min((first >> 5) + it * 8u, (uint32_t)H * W - 1), 256, g * 8, v[it]);
#pragma unroll
    for (int it = 0; it < kIt; ++it) {
        const uint32_t i = first + it * 256u;
        if (i >= items) break;
        const int hw = (int)(i >> 5);
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[j] = (v[it][j] - mu) * rstd * ga[j] + be[j];
            if (P.relu) o[j] = fmaxf(o[j], 0.f);
        }
        if (pr.up) {
            const int h = hw / W, w = hw - h * W;
            float t[8];
            Act<SPLIT>::ld8(pr.up, up_img + (size_t)((h * Hu) / H) * Wu + (w * Wu) / W, 256, g * 8, t);
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] += t[j];
        }
        Act<SPLIT>::st8(pr.y, img + hw, 256, g * 8, o);
    }
}

// Space-to-depth form of the stem input: v[n][Y][X][(dy*2+dx)*3 + c] = img[n][c][2(Y-2)+dy][2(X-2)+dx] (zero outside
// the image, channels 12-15 zero), Y in [0, H/2+3), X in [0, W/2+3).  conv1 (7x7, stride 2, pad 3; resnet.py:495)
// is then a 4x4 stride-1 convolution over 16 channels, which the tensor-core kernel reads straight through TMA.
// bf16: interleaved [N,Hp,Wp,16].  Split: two planes [2][N,Hp,Wp,16] (hi plane, then lo plane).
// SRC_U8: the decoded image as the data pipeline holds it, uint8 HWC [N,H,W,3] (cv2 channel order).  The Normalize step
// of the test pipeline (mmdet/datasets/pipelines/transforms.py Normalize -> mmcv.imnormalize: optional BGR->RGB,
// (x - mean) * (1/std) in fp32) is applied on the fly, so a step uploads 3 bytes per pixel instead of 12.  mean / stdinv
// are indexed by MODEL channel c; model channel c is image channel (to_rgb ? 2-c : c).  valid (SRC_U8 only; int32 [N,2]
// = (h, w) per image, or null for the full extent): pixels at y >= h or x >= w are the Pad step that follows Normalize
// in the pipeline and contribute exactly 0.0.
template <bool SPLIT, bool SRC_U8>
__global__ void __launch_bounds__(256)
stem_s2d_kernel(const void *__restrict__ img_v, int N, int H, int W, float3 mean, float3 stdinv, int to_rgb,
                const int32_t *__restrict__ valid, typename Act<SPLIT>::T *__restrict__ out)
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
        const long long lo = (long long)total * 16;                           // split: offset of the lo plane
        Act<SPLIT>::st8(out + i * 16, lo, v0);
        Act<SPLIT>::st8(out + i * 16 + 8, lo, v1);
    }
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
        Act<true>::st8(y, pix, C, c, v);
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
        Act<true>::ld8(x, pix, C, c, v);
        *reinterpret_cast<float4 *>(y + pix * C + c) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4 *>(y + pix * C + c + 4) = make_float4(v[4], v[5], v[6], v[7]);
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
            if (MODE == 0)
                static_cast<float *>(yv)[(size_t)n * R * Cc + (size_t)c * R + r] = v;
            else
                Act<true>::st(static_cast<__half *>(yv), (long long)n * Cc + c, R, r, v);   // pixel c: [2][R channels]
        }
    }
}

// ---- DCNv2 backbone convolutions (deform_conv.py:411-419): conv_offset output [pixels, 27] -> offset [pixels, 18] (channels
// 0..17 as they are: cat(o1, o2)) and mask [pixels, 9] = sigmoid(channels 18..26).  One element per thread, both sides
// coalesced.  The sigmoid is taken in fp64 and rounded once, so the mask is the correctly rounded fp32 value up to the
// fp64 exp's error.
__global__ void __launch_bounds__(256)
dcnv2_offset_mask_kernel(const float *__restrict__ om, size_t pixels, float *__restrict__ offset, float *__restrict__ mask)
{
    const size_t total = pixels * 27;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / 27;
        const int c = (int)(i - pix * 27);
        const float v = om[i];
        if (c < 18) offset[pix * 18 + c] = v;
        else mask[pix * 9 + (c - 18)] = (float)(1.0 / (1.0 + exp(-(double)v)));
    }
}

}  // namespace
}  // namespace orp

using namespace orp;

template <bool SPLIT, bool SRC_U8>
static int stem_s2d_impl(const void *img, int N, int H, int W, const float *mean, const float *std, int to_rgb,
                         const int32_t *valid, void *out, void *stream)
{
    if (!img || !out || (SRC_U8 && (!mean || !std)) || N < 1 || H < 2 || W < 2 || (H & 1) || (W & 1))
        return fail(ORP_EINVAL, SRC_U8 ? "stem_s2d_u8_%s: needs even H, W" : "stem_s2d_%s: needs even H, W", fmt_name(SPLIT));
    int rc = ensure_device();
    if (rc) return rc;
    float3 mu = make_float3(0.f, 0.f, 0.f), si = mu;
    if (SRC_U8) {
        mu = make_float3(mean[0], mean[1], mean[2]);
        // mmcv.imnormalize: stdinv = 1 / np.float64(std), applied to the float32 image
        si = make_float3((float)(1.0 / (double)std[0]), (float)(1.0 / (double)std[1]), (float)(1.0 / (double)std[2]));
    }
    const size_t total = (size_t)N * (H / 2 + 3) * (W / 2 + 3);
    stem_s2d_kernel<SPLIT, SRC_U8><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img, N, H, W, mu, si, to_rgb, valid, static_cast<typename Act<SPLIT>::T *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_stem_s2d_bf16(const float *img_nchw, int N, int H, int W, void *out, void *stream)
{
    return stem_s2d_impl<false, false>(img_nchw, N, H, W, nullptr, nullptr, 0, nullptr, out, stream);
}

extern "C" int orp_stem_s2d_f16x3(const float *img_nchw, int N, int H, int W, void *out, void *stream)
{
    return stem_s2d_impl<true, false>(img_nchw, N, H, W, nullptr, nullptr, 0, nullptr, out, stream);
}

extern "C" int orp_stem_s2d_u8_bf16(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                    int to_rgb, void *out, void *stream)
{
    return stem_s2d_impl<false, true>(img_hwc, N, H, W, mean, std, to_rgb, nullptr, out, stream);
}

extern "C" int orp_stem_s2d_u8_f16x3(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                     int to_rgb, void *out, void *stream)
{
    return stem_s2d_impl<true, true>(img_hwc, N, H, W, mean, std, to_rgb, nullptr, out, stream);
}

extern "C" int orp_stem_s2d_u8_padded_bf16(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                           int to_rgb, const int32_t *valid_hw, void *out, void *stream)
{
    if (!valid_hw) return fail(ORP_EINVAL, "stem_s2d_u8_padded_bf16: valid_hw is required");
    return stem_s2d_impl<false, true>(img_hwc, N, H, W, mean, std, to_rgb, valid_hw, out, stream);
}

extern "C" int orp_stem_s2d_u8_padded_f16x3(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                            int to_rgb, const int32_t *valid_hw, void *out, void *stream)
{
    if (!valid_hw) return fail(ORP_EINVAL, "stem_s2d_u8_padded_f16x3: valid_hw is required");
    return stem_s2d_impl<true, true>(img_hwc, N, H, W, mean, std, to_rgb, valid_hw, out, stream);
}

extern "C" int orp_stem_im2col_bf16(const float *img_nchw, int N, int H, int W, void *out, void *stream)
{
    if (!img_nchw || !out || N <= 0) return fail(ORP_EINVAL, "stem_im2col_bf16: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
    const int wblocks = (Wo + kStemPix - 1) / kStemPix;
    stem_im2col_kernel<<<(unsigned)((size_t)N * Ho * wblocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img_nchw, N, H, W, Ho, Wo, static_cast<__nv_bfloat16 *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}

template <bool SPLIT>
static int maxpool3x3s2_impl(const void *x, int N, int H, int W, int C, void *y, void *stream)
{
    typedef typename Act<SPLIT>::T T;
    if (!x || !y || C % 8) return fail(ORP_EINVAL, "maxpool3x3s2_%s: bad arguments", fmt_name(SPLIT));
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const size_t total = (size_t)N * Ho * Wo * (C / 8);
    maxpool3x3s2_kernel<SPLIT><<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const T *>(x), N, H, W, C, Ho, Wo, static_cast<T *>(y));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_maxpool3x3s2_bf16(const void *x, int N, int H, int W, int C, void *y, void *stream)
{
    return maxpool3x3s2_impl<false>(x, N, H, W, C, y, stream);
}

extern "C" int orp_maxpool3x3s2_f16x3(const void *x, int N, int H, int W, int C, void *y, void *stream)
{
    return maxpool3x3s2_impl<true>(x, N, H, W, C, y, stream);
}

template <bool SPLIT>
static int gn_stats_impl(const void *x, int N, int HW, int C, int groups, double *stats, void *stream)
{
    if (!x || !stats || C != 256 || groups != 32) return fail(ORP_EINVAL, "gn_stats_%s: needs C=256, 32 groups", fmt_name(SPLIT));
    int rc = ensure_device();
    if (rc) return rc;
    int slabs = ceil_div(HW, 64);
    const int maxs = (kNumSMs * 4 + N - 1) / N;
    if (slabs > maxs) slabs = maxs;
    const int slab = ceil_div(HW, slabs);
    slabs = ceil_div(HW, slab);
    gn_stats_kernel<SPLIT><<<dim3(slabs, N), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const typename Act<SPLIT>::T *>(x), HW, slab, stats);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_stats_bf16(const void *x, int N, int HW, int C, int groups, double *stats, void *stream)
{
    return gn_stats_impl<false>(x, N, HW, C, groups, stats, stream);
}

extern "C" int orp_gn_stats_f16x3(const void *x, int N, int HW, int C, int groups, double *stats, void *stream)
{
    return gn_stats_impl<true>(x, N, HW, C, groups, stats, stream);
}

template <bool SPLIT>
static int gn_apply_multi_impl(int nprob, const orp_gn_problem *probs, int C, int groups, const float *gamma, const float *beta,
                               float eps, int relu, void *stream)
{
    typedef typename Act<SPLIT>::T T;
    const char *name = fmt_name(SPLIT);
    if (nprob < 1 || nprob > 8 || !probs || !gamma || !beta || C != 256 || groups != 32)
        return fail(ORP_EINVAL, "gn_apply_%s: needs 1..8 problems, C=256, 32 groups", name);
    int rc = ensure_device();
    if (rc) return rc;
    GnApplyParams<T> P;
    memset(&P, 0, sizeof(P));
    P.nprob = nprob; P.gamma = gamma; P.beta = beta; P.eps = eps; P.relu = relu;
    int imgs = 0;
    size_t max_items = 0;
    for (int i = 0; i < nprob; ++i) {
        const orp_gn_problem &q = probs[i];
        if (!q.x || !q.y || !q.stats || q.N < 1 || q.H < 1 || q.W < 1) return fail(ORP_EINVAL, "gn_apply_%s: bad problem", name);
        if ((size_t)q.H * q.W * 32 > 0xffffffffull) return fail(ORP_EINVAL, "gn_apply_%s: image too large", name);
        P.p[i].x = static_cast<const T *>(q.x);
        P.p[i].stats = q.stats;
        P.p[i].up = static_cast<const T *>(q.up_src);
        P.p[i].y = static_cast<T *>(q.y);
        P.p[i].N = q.N; P.p[i].H = q.H; P.p[i].W = q.W;
        P.p[i].img_start = imgs;
        imgs += q.N;
        const size_t c = (size_t)q.H * q.W * 32;
        max_items = c > max_items ? c : max_items;
    }
    if (imgs > 65535) return fail(ORP_EINVAL, "gn_apply_%s: too many images", name);
    constexpr unsigned kBlockItems = kGnApplyIt<SPLIT> * 256;
    dim3 grid((unsigned)((max_items + kBlockItems - 1) / kBlockItems), (unsigned)imgs);
    gn_apply_kernel<SPLIT><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_apply_bf16_multi(int nprob, const orp_gn_problem *probs, int C, int groups, const float *gamma,
                                       const float *beta, float eps, int relu, void *stream)
{
    return gn_apply_multi_impl<false>(nprob, probs, C, groups, gamma, beta, eps, relu, stream);
}

extern "C" int orp_gn_apply_f16x3_multi(int nprob, const orp_gn_problem *probs, int C, int groups, const float *gamma,
                                        const float *beta, float eps, int relu, void *stream)
{
    return gn_apply_multi_impl<true>(nprob, probs, C, groups, gamma, beta, eps, relu, stream);
}

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

extern "C" int orp_dcnv2_offset_mask(const float *om, long long pixels, float *offset, float *mask, void *stream)
{
    if (!om || !offset || !mask || pixels < 0) return fail(ORP_EINVAL, "dcnv2_offset_mask: bad arguments");
    if (pixels == 0) return ORP_OK;
    int rc = ensure_device();
    if (rc) return rc;
    dcnv2_offset_mask_kernel<<<grid_for((size_t)pixels * 27, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        om, (size_t)pixels, offset, mask);
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
