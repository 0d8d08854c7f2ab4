// dense_bf16_misc.cu - the memory-bound companions of the tensor-core convolutions (NHWC bf16):
// stem im2col (7x7/2, 3 channels -> one 192-wide K block row per output pixel), 3x3/2 max-pool,
// GroupNorm statistics and apply (+ReLU, + the FPN top-down nearest-2x add).  All HBM-bound: 16-byte
// vector accesses, grids sized in multiples of the SM count.
#include <cuda_bf16.h>
#include <cstring>

#include "common.cuh"

namespace orp {
namespace {

__device__ __forceinline__ uint32_t pack2(float a, float b)
{
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&v);
}
__device__ __forceinline__ float2 unpack2(uint32_t u)
{
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u));
}

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
        *reinterpret_cast<uint4 *>(orow + (size_t)item * 8) = make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
    }
}

__global__ void __launch_bounds__(256)
maxpool3x3s2_bf16_kernel(const __nv_bfloat16 *__restrict__ x, int N, int H, int W, int C, int Ho, int Wo,
                         __nv_bfloat16 *__restrict__ y)
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
                const uint4 u = *reinterpret_cast<const uint4 *>(x + (((size_t)n * H + ih) * W + iw) * C + c);
                const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 f = unpack2(uu[k]);
                    m[2 * k] = fmaxf(m[2 * k], f.x);
                    m[2 * k + 1] = fmaxf(m[2 * k + 1], f.y);
                }
            }
        *reinterpret_cast<uint4 *>(y + pix * C + c) = make_uint4(pack2(m[0], m[1]), pack2(m[2], m[3]), pack2(m[4], m[5]), pack2(m[6], m[7]));
    }
}

// GroupNorm statistics of a bf16 NHWC tensor with C = 256, 32 groups (8 channels = one 16-byte vector
// = one lane): grid (slabs, N); every warp strides over the pixels of its slab, lane l owns group l.
__global__ void __launch_bounds__(256)
gn_stats_bf16_kernel(const __nv_bfloat16 *__restrict__ x, int HW, int slab, double *__restrict__ stats)
{
    __shared__ float s_sum[8][32], s_sq[8][32];
    const int n = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int p0 = blockIdx.x * slab, p1 = min(HW, p0 + slab);
    const __nv_bfloat16 *base = x + (size_t)n * HW * 256 + lane * 8;
    float s = 0.f, q = 0.f;
    for (int p = p0 + warp; p < p1; p += 8) {
        const uint4 u = *reinterpret_cast<const uint4 *>(base + (size_t)p * 256);
        const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = unpack2(uu[k]);
            s += f.x + f.y;
            q += f.x * f.x + f.y * f.y;
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

struct GnApplyProb {
    const __nv_bfloat16 *x;
    const double *stats;
    const __nv_bfloat16 *up;
    __nv_bfloat16 *y;
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

// One (problem, image) per blockIdx.y.  A thread always works on the same channel group (its index & 31), so the
// group's mean / rstd and the eight gamma / beta values live in registers; per 16-byte chunk the work is one load,
// eight multiply-adds, the optional nearest-neighbour top-down add (fpn.py:171-176) and one store.
__global__ void __launch_bounds__(256)
gn_apply_bf16_kernel(const __grid_constant__ GnApplyParams P)
{
    int pi = 0;
#pragma unroll
    for (int k = 1; k < 8; ++k)
        if (k < P.nprob && (int)blockIdx.y >= P.p[k].img_start) pi = k;
    const GnApplyProb &pr = P.p[pi];
    const int n = (int)blockIdx.y - pr.img_start;
    const int H = pr.H, W = pr.W;
    const uint32_t chunks = (uint32_t)H * W * 32;           // 16-byte chunks of this image
    const uint32_t first = blockIdx.x * 2048u + threadIdx.x;
    if (first >= chunks) return;
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
    const uint4 *xi = reinterpret_cast<const uint4 *>(pr.x) + (size_t)n * chunks;
    uint4 *yi = reinterpret_cast<uint4 *>(pr.y) + (size_t)n * chunks;
    const int Hu = (H + 1) / 2, Wu = (W + 1) / 2;           // F.interpolate(size=prev_shape, mode='nearest'): src = floor(dst * in / out)
    const __nv_bfloat16 *upi = pr.up ? pr.up + (size_t)n * Hu * Wu * 256 + g * 8 : nullptr;
    uint4 u[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const uint32_t i = first + it * 256u;
        if (i < chunks) u[it] = xi[i];
    }
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const uint32_t i = first + it * 256u;
        if (i >= chunks) break;
        const uint32_t uu[4] = {u[it].x, u[it].y, u[it].z, u[it].w};
        float o[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = unpack2(uu[k]);
            o[2 * k] = f.x;
            o[2 * k + 1] = f.y;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[j] = (o[j] - mu) * rstd * ga[j] + be[j];
            if (P.relu) o[j] = fmaxf(o[j], 0.f);
        }
        if (upi) {
            const int hw = (int)(i >> 5);
            const int h = hw / W, w = hw - h * W;
            const uint4 v = *reinterpret_cast<const uint4 *>(upi + ((size_t)((h * Hu) / H) * Wu + (w * Wu) / W) * 256);
            const uint32_t vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 f = unpack2(vv[k]);
                o[2 * k] += f.x;
                o[2 * k + 1] += f.y;
            }
        }
        yi[i] = make_uint4(pack2(o[0], o[1]), pack2(o[2], o[3]), pack2(o[4], o[5]), pack2(o[6], o[7]));
    }
}

int grid_for(size_t items, int threads)
{
    size_t g = (items + threads - 1) / threads;
    const size_t cap = kNumSMs * 16;
    return (int)(g < cap ? (g ? g : 1) : cap);
}

}  // namespace
}  // namespace orp

using namespace orp;

namespace orp {
namespace {
// Space-to-depth form of the stem input: out[n][Y][X][(dy*2+dx)*3 + c] = img[n][c][2(Y-2)+dy][2(X-2)+dx] (zero outside
// the image, channels 12-15 zero), Y in [0, H/2+3), X in [0, W/2+3).  conv1 (7x7, stride 2, pad 3; resnet.py:495)
// is then a 4x4 stride-1 convolution over 16 channels, which the tensor-core kernel reads straight through TMA.
__global__ void __launch_bounds__(256)
stem_s2d_kernel(const float *__restrict__ img, int N, int H, int W, __nv_bfloat16 *__restrict__ out)
{
    const int Hp = H / 2 + 3, Wp = W / 2 + 3;
    const size_t total = (size_t)N * Hp * Wp;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int X = (int)(i % Wp);
        const size_t t = i / Wp;
        const int Y = (int)(t % Hp), n = (int)(t / Hp);
        const int y0 = 2 * (Y - 2), x0 = 2 * (X - 2);
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = 0.f;
        if (x0 >= 0 && x0 + 1 < W) {
#pragma unroll
            for (int dy = 0; dy < 2; ++dy) {
                const int y = y0 + dy;
                if (y < 0 || y >= H) continue;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const float2 p = *reinterpret_cast<const float2 *>(img + (((size_t)n * 3 + c) * H + y) * W + x0);
                    v[(dy * 2 + 0) * 3 + c] = p.x;
                    v[(dy * 2 + 1) * 3 + c] = p.y;
                }
            }
        }
        uint4 o0 = make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
        uint4 o1 = make_uint4(pack2(v[8], v[9]), pack2(v[10], v[11]), pack2(v[12], v[13]), pack2(v[14], v[15]));
        uint4 *op = reinterpret_cast<uint4 *>(out + i * 16);
        op[0] = o0;
        op[1] = o1;
    }
}

// The same from the decoded image as the data pipeline holds it: uint8 HWC [N,H,W,3] (cv2 channel order).  The
// Normalize step of the test pipeline (mmdet/datasets/pipelines/transforms.py Normalize -> mmcv.imnormalize:
// optional BGR->RGB, (x - mean) * (1/std) in fp32) is applied on the fly, so a step uploads 3 bytes per pixel
// instead of 12.  mean / stdinv are indexed by MODEL channel c; model channel c is image channel (to_rgb ? 2-c : c).
// valid (int32 [N,2] = (h, w) per image, or null for the full extent): pixels at y >= h or x >= w are the Pad step
// that follows Normalize in the pipeline and contribute exactly 0.0.
__global__ void __launch_bounds__(256)
stem_s2d_u8_kernel(const uint8_t *__restrict__ img, int N, int H, int W, float3 mean, float3 stdinv, int to_rgb,
                   const int32_t *__restrict__ valid, __nv_bfloat16 *__restrict__ out)
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
        if (x0 >= 0 && x0 < vw) {
#pragma unroll
            for (int dy = 0; dy < 2; ++dy) {
                const int y = y0 + dy;
                if (y < 0 || y >= vh) continue;
                const uint8_t *p = img + (((size_t)n * H + y) * W + x0) * 3;     // 6 bytes: two pixels (W is even)
                // x0 even -> the 6 bytes start at an even address
                const uint16_t a = *reinterpret_cast<const uint16_t *>(p), b = *reinterpret_cast<const uint16_t *>(p + 2),
                               c2 = *reinterpret_cast<const uint16_t *>(p + 4);
                const uint8_t px[6] = {(uint8_t)(a & 0xff), (uint8_t)(a >> 8), (uint8_t)(b & 0xff), (uint8_t)(b >> 8),
                                       (uint8_t)(c2 & 0xff), (uint8_t)(c2 >> 8)};
#pragma unroll
                for (int dx = 0; dx < 2; ++dx) {
                    if (x0 + dx >= vw) continue;                              // odd valid width: the pair's second pixel is padding
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const int sc = to_rgb ? 2 - c : c;
                        v[(dy * 2 + dx) * 3 + c] = ((float)px[dx * 3 + sc] - mu[c]) * si[c];
                    }
                }
            }
        }
        uint4 o0 = make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
        uint4 o1 = make_uint4(pack2(v[8], v[9]), pack2(v[10], v[11]), pack2(v[12], v[13]), pack2(v[14], v[15]));
        uint4 *op = reinterpret_cast<uint4 *>(out + i * 16);
        op[0] = o0;
        op[1] = o1;
    }
}
}  // namespace
}  // namespace orp

static int stem_s2d_u8_bf16_impl(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std, int to_rgb,
                                 const int32_t *valid, void *out, void *stream)
{
    using namespace orp;
    if (!img_hwc || !out || !mean || !std || N < 1 || H < 2 || W < 2 || (H & 1) || (W & 1))
        return fail(ORP_EINVAL, "stem_s2d_u8_bf16: needs even H, W");
    int rc = ensure_device();
    if (rc) return rc;
    const float3 mu = make_float3(mean[0], mean[1], mean[2]);
    // mmcv.imnormalize: stdinv = 1 / np.float64(std), applied to the float32 image
    const float3 si = make_float3((float)(1.0 / (double)std[0]), (float)(1.0 / (double)std[1]), (float)(1.0 / (double)std[2]));
    const size_t total = (size_t)N * (H / 2 + 3) * (W / 2 + 3);
    stem_s2d_u8_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(img_hwc, N, H, W, mu, si, to_rgb, valid,
                                                                                           static_cast<__nv_bfloat16 *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_stem_s2d_u8_bf16(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                    int to_rgb, void *out, void *stream)
{
    return stem_s2d_u8_bf16_impl(img_hwc, N, H, W, mean, std, to_rgb, nullptr, out, stream);
}

extern "C" int orp_stem_s2d_u8_padded_bf16(const uint8_t *img_hwc, int N, int H, int W, const float *mean, const float *std,
                                           int to_rgb, const int32_t *valid_hw, void *out, void *stream)
{
    if (!valid_hw) return orp::fail(ORP_EINVAL, "stem_s2d_u8_padded_bf16: valid_hw is required");
    return stem_s2d_u8_bf16_impl(img_hwc, N, H, W, mean, std, to_rgb, valid_hw, out, stream);
}

extern "C" int orp_stem_s2d_bf16(const float *img_nchw, int N, int H, int W, void *out, void *stream)
{
    using namespace orp;
    if (!img_nchw || !out || N < 1 || H < 2 || W < 2 || (H & 1) || (W & 1)) return fail(ORP_EINVAL, "stem_s2d_bf16: needs even H, W");
    int rc = ensure_device();
    if (rc) return rc;
    const size_t total = (size_t)N * (H / 2 + 3) * (W / 2 + 3);
    stem_s2d_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(img_nchw, N, H, W,
                                                                                        static_cast<__nv_bfloat16 *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
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

extern "C" int orp_maxpool3x3s2_bf16(const void *x, int N, int H, int W, int C, void *y, void *stream)
{
    if (!x || !y || C % 8) return fail(ORP_EINVAL, "maxpool3x3s2_bf16: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const size_t total = (size_t)N * Ho * Wo * (C / 8);
    maxpool3x3s2_bf16_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16 *>(x), N, H, W, C, Ho, Wo, static_cast<__nv_bfloat16 *>(y));
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_stats_bf16(const void *x, int N, int HW, int C, int groups, double *stats, void *stream)
{
    if (!x || !stats || C != 256 || groups != 32) return fail(ORP_EINVAL, "gn_stats_bf16: needs C=256, 32 groups");
    int rc = ensure_device();
    if (rc) return rc;
    int slabs = ceil_div(HW, 64);
    const int maxs = (kNumSMs * 4 + N - 1) / N;
    if (slabs > maxs) slabs = maxs;
    const int slab = ceil_div(HW, slabs);
    slabs = ceil_div(HW, slab);
    gn_stats_bf16_kernel<<<dim3(slabs, N), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16 *>(x), HW, slab, stats);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_apply_bf16_multi(int nprob, const orp_gn_problem *probs, int C, int groups, const float *gamma,
                                       const float *beta, float eps, int relu, void *stream)
{
    if (nprob < 1 || nprob > 8 || !probs || !gamma || !beta || C != 256 || groups != 32)
        return fail(ORP_EINVAL, "gn_apply_bf16: needs 1..8 problems, C=256, 32 groups");
    int rc = ensure_device();
    if (rc) return rc;
    GnApplyParams P;
    memset(&P, 0, sizeof(P));
    P.nprob = nprob; P.gamma = gamma; P.beta = beta; P.eps = eps; P.relu = relu;
    int imgs = 0;
    size_t max_chunks = 0;
    for (int i = 0; i < nprob; ++i) {
        const orp_gn_problem &q = probs[i];
        if (!q.x || !q.y || !q.stats || q.N < 1 || q.H < 1 || q.W < 1) return fail(ORP_EINVAL, "gn_apply_bf16: bad problem");
        if ((size_t)q.H * q.W * 32 > 0xffffffffull) return fail(ORP_EINVAL, "gn_apply_bf16: image too large");
        P.p[i].x = static_cast<const __nv_bfloat16 *>(q.x);
        P.p[i].stats = q.stats;
        P.p[i].up = static_cast<const __nv_bfloat16 *>(q.up_src);
        P.p[i].y = static_cast<__nv_bfloat16 *>(q.y);
        P.p[i].N = q.N; P.p[i].H = q.H; P.p[i].W = q.W;
        P.p[i].img_start = imgs;
        imgs += q.N;
        const size_t c = (size_t)q.H * q.W * 32;
        max_chunks = c > max_chunks ? c : max_chunks;
    }
    if (imgs > 65535) return fail(ORP_EINVAL, "gn_apply_bf16: too many images");
    dim3 grid((unsigned)((max_chunks + 2047) / 2048), (unsigned)imgs);
    gn_apply_bf16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_apply_bf16(const void *x, int N, int H, int W, int C, const double *stats, int groups,
                                 const float *gamma, const float *beta, float eps, int relu, const void *up_src, void *y,
                                 void *stream)
{
    orp_gn_problem q;
    q.x = x; q.N = N; q.H = H; q.W = W; q.stats = stats; q.up_src = up_src; q.y = y;
    return orp_gn_apply_bf16_multi(1, &q, C, groups, gamma, beta, eps, relu, stream);
}
