// dense_f32.cu - fp32 (CUDA-core) dense layers of the OrientedRepPoints inference path, NHWC.
//
// The CUDA-core mirror of the reference's fp32 arithmetic: plain fp32 multiply-adds like its fp32
// cuDNN/cuBLAS convolutions (mmdet/models/backbones/resnet.py:203-239,495-506,
// necks/fpn.py:138-178, anchor_heads/orientedreppoints_head.py:148-171) and its deformable im2col +
// SGEMM (mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:84-115,190-243, deform_conv_cuda.cpp:152-260).
// ReLU and max-pool propagate NaN as nn.ReLU / nn.MaxPool2d do.  It is the detector's default
// precision and the reference engine of several GPU tests; the benchmarked parity arithmetic is
// f16x3 on the tensor cores (dense_tc.cu), which tests compare with this engine and with fp64.
//
// One implicit-GEMM kernel serves ordinary and deformable convolutions: M = output pixels of one
// image (tiles never straddle images), N = output channels, K = taps x input channels; the
// deformable variant replaces the A-operand load by the reference's 4-corner bilinear sample, so
// the 151 MB `columns` scratch of the reference (2304 x H*W floats at stride 8) never exists.
// Epilogue fuses bias, residual add, ReLU and the per-(image, group) sum / sum-of-squares that
// GroupNorm needs (fp32 partials per thread and per CTA, added across CTAs with double atomics).
#include "common.cuh"
#include "../../include/orp_b200_group.h"
#include "../../include/orp_b200_hrnet.h"
#include "hrnet.cuh"

namespace orp {
namespace {

// max(a, b) that returns a NaN operand, as torch's max-pool and ReLU do (fmaxf drops it)
__device__ __forceinline__ float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }

struct ConvP {
    const float *x, *w, *bias, *res, *off, *mask;
    float *y;
    double *stats;
    int N, H, W, Cin, Cout, KH, KW, stride, pad, dil, Ho, Wo, K, relu, groups, tiles_per_img;
};

constexpr int BM = 128, BN = 64, BK = 16;

template <bool DEFORM>
__device__ __forceinline__ float4 load_a(const ConvP &p, int n, int oh, int ow, bool row_ok, int k)
{
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!row_ok || k >= p.K) return v;
    const int tap = k / p.Cin, ci = k - tap * p.Cin;
    const int kh = tap / p.KW, kw = tap - kh * p.KW;
    const int hb = oh * p.stride - p.pad + kh * p.dil, wb = ow * p.stride - p.pad + kw * p.dil;
    const float *img = p.x + (size_t)n * p.H * p.W * p.Cin;
    if (!DEFORM) {
        if (hb >= 0 && hb < p.H && wb >= 0 && wb < p.W)
            v = *reinterpret_cast<const float4 *>(img + ((size_t)hb * p.W + wb) * p.Cin + ci);
        return v;
    }
    // deformable_im2col_gpu_kernel: offsets (dy, dx) interleaved per tap, NHWC here
    const float *o = p.off + (((size_t)n * p.Ho + oh) * p.Wo + ow) * (2 * p.KH * p.KW) + 2 * tap;
    const float h_im = (float)hb + o[0], w_im = (float)wb + o[1];
    if (!(h_im > -1.f && w_im > -1.f && h_im < (float)p.H && w_im < (float)p.W)) return v;
    const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
    const int h_high = h_low + 1, w_high = w_low + 1;
    const float lh = h_im - (float)h_low, lw = w_im - (float)w_low, hh = 1.f - lh, hw = 1.f - lw;
    float4 v1 = v, v2 = v, v3 = v, v4 = v;
    if (h_low >= 0 && w_low >= 0) v1 = *reinterpret_cast<const float4 *>(img + ((size_t)h_low * p.W + w_low) * p.Cin + ci);
    if (h_low >= 0 && w_high <= p.W - 1) v2 = *reinterpret_cast<const float4 *>(img + ((size_t)h_low * p.W + w_high) * p.Cin + ci);
    if (h_high <= p.H - 1 && w_low >= 0) v3 = *reinterpret_cast<const float4 *>(img + ((size_t)h_high * p.W + w_low) * p.Cin + ci);
    if (h_high <= p.H - 1 && w_high <= p.W - 1) v4 = *reinterpret_cast<const float4 *>(img + ((size_t)h_high * p.W + w_high) * p.Cin + ci);
    const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
    float m = 1.f;
    if (p.mask) m = p.mask[(((size_t)n * p.Ho + oh) * p.Wo + ow) * (p.KH * p.KW) + tap];   // DCNv2 modulation
    v.x = (w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x) * m;
    v.y = (w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y) * m;
    v.z = (w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z) * m;
    v.w = (w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w) * m;
    return v;
}

template <bool DEFORM>
__global__ void __launch_bounds__(256)
conv_f32_kernel(ConvP p)
{
    __shared__ float As[2][BK][BM];
    __shared__ float Bs[2][BK][BN];
    __shared__ float s_sum[BN], s_sq[BN];
    const int t = threadIdx.x;
    const int n = blockIdx.x / p.tiles_per_img;
    const int tile = blockIdx.x - n * p.tiles_per_img;
    const int m0 = tile * BM, n0 = blockIdx.y * BN;
    const int HoWo = p.Ho * p.Wo;

    // A loader: two (row, quarter) items per thread; rows are consecutive across threads
    int a_m[2], a_q[2], a_oh[2], a_ow[2];
    bool a_ok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int item = t + i * 256;
        a_m[i] = item & (BM - 1);
        a_q[i] = item >> 7;
        const int pix = m0 + a_m[i];
        a_ok[i] = pix < HoWo;
        a_oh[i] = a_ok[i] ? pix / p.Wo : 0;
        a_ow[i] = a_ok[i] ? pix - a_oh[i] * p.Wo : 0;
    }
    const int b_n = t & (BN - 1), b_q = t >> 6;
    const bool b_ok = (n0 + b_n) < p.Cout;
    const float *wrow = p.w + (size_t)(n0 + b_n) * p.K;

    const int ty = t >> 4, tx = t & 15;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int nk = (p.K + BK - 1) / BK;
    float4 ra[2], rb;
    auto gload = [&](int kc) {
#pragma unroll
        for (int i = 0; i < 2; ++i) ra[i] = load_a<DEFORM>(p, n, a_oh[i], a_ow[i], a_ok[i], kc * BK + a_q[i] * 4);
        const int k = kc * BK + b_q * 4;
        rb = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b_ok && k < p.K) rb = *reinterpret_cast<const float4 *>(wrow + k);   // K % 4 == 0
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            As[buf][a_q[i] * 4 + 0][a_m[i]] = ra[i].x;
            As[buf][a_q[i] * 4 + 1][a_m[i]] = ra[i].y;
            As[buf][a_q[i] * 4 + 2][a_m[i]] = ra[i].z;
            As[buf][a_q[i] * 4 + 3][a_m[i]] = ra[i].w;
        }
        Bs[buf][b_q * 4 + 0][b_n] = rb.x;
        Bs[buf][b_q * 4 + 1][b_n] = rb.y;
        Bs[buf][b_q * 4 + 2][b_n] = rb.z;
        Bs[buf][b_q * 4 + 3][b_n] = rb.w;
    };
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kc = 0; kc < nk; ++kc) {
        const int buf = kc & 1;
        if (kc + 1 < nk) gload(kc + 1);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * 8 + 4]);
            const float4 b = *reinterpret_cast<const float4 *>(&Bs[buf][kk][tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        if (kc + 1 < nk) sstore(buf ^ 1);
        __syncthreads();
    }

    // ------------------------------------------------------------------ epilogue
    const bool want_stats = p.stats != nullptr;
    if (want_stats) {
        if (t < BN) { s_sum[t] = 0.f; s_sq[t] = 0.f; }
        __syncthreads();
    }
    float csum[4] = {0.f, 0.f, 0.f, 0.f}, csq[4] = {0.f, 0.f, 0.f, 0.f};
    const int cb = n0 + tx * 4;
    const bool vec_ok = ((p.Cout & 3) == 0) && (cb + 3 < p.Cout);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int pix = m0 + ty * 8 + i;
        if (pix >= HoWo) continue;
        const size_t base = ((size_t)n * HoWo + pix) * p.Cout + cb;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[j] = acc[i][j];
            if (p.bias && cb + j < p.Cout) v[j] += p.bias[cb + j];
        }
        if (p.res) {
            if (vec_ok) {
                const float4 r = *reinterpret_cast<const float4 *>(p.res + base);
                v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j) if (cb + j < p.Cout) v[j] += p.res[base + j];
            }
        }
        if (p.relu) {
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = max_nan(v[j], 0.f);
        }
        if (vec_ok) {
            *reinterpret_cast<float4 *>(p.y + base) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (cb + j < p.Cout) p.y[base + j] = v[j];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { csum[j] += v[j]; csq[j] += v[j] * v[j]; }
    }
    if (want_stats) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            atomicAdd(&s_sum[tx * 4 + j], csum[j]);
            atomicAdd(&s_sq[tx * 4 + j], csq[j]);
        }
        __syncthreads();
        if (t < BN && n0 + t < p.Cout) {
            const int g = (n0 + t) / (p.Cout / p.groups);
            atomicAdd(&p.stats[((size_t)n * p.groups + g) * 2 + 0], (double)s_sum[t]);
            atomicAdd(&p.stats[((size_t)n * p.groups + g) * 2 + 1], (double)s_sq[t]);
        }
    }
}

// Grouped 3x3 convolution, pad 1 (ResNeXt conv2, resnext.py:44-54): one thread per output pixel and 4 consecutive output
// channels, which share a group (gw % 4 == 0).  Each sums the 9 gw products of its group in the implicit GEMM's order (taps,
// then input channels), float4 reads of x and of the weights [C][3][3][gw].
__global__ void __launch_bounds__(256)
group_conv3x3_f32_kernel(const float *__restrict__ x, int N, int H, int W, int C, int gw, const float *__restrict__ w, int stride,
                         int Ho, int Wo, const float *__restrict__ bias, int relu, float *__restrict__ y)
{
    const int c4n = C / 4;
    const size_t total = (size_t)N * Ho * Wo * c4n;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / c4n;
        const int co = (int)(i - pix * c4n) * 4;
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), n = (int)(pix / ((size_t)Wo * Ho));
        const int ci0 = co - co % gw;                             // first input channel of the group
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int kh = 0; kh < 3; ++kh) {
            const int ih = oh * stride - 1 + kh;
            if (ih < 0 || ih >= H) continue;
            for (int kw = 0; kw < 3; ++kw) {
                const int iw = ow * stride - 1 + kw;
                if (iw < 0 || iw >= W) continue;
                const float *xp = x + (((size_t)n * H + ih) * W + iw) * C + ci0;
                const float *wp = w + ((size_t)co * 9 + kh * 3 + kw) * gw;
                for (int c = 0; c < gw; c += 4) {
                    const float4 xv = *reinterpret_cast<const float4 *>(xp + c);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float4 wv = *reinterpret_cast<const float4 *>(wp + (size_t)j * 9 * gw + c);
                        acc[j] = fmaf(xv.x, wv.x, acc[j]);
                        acc[j] = fmaf(xv.y, wv.y, acc[j]);
                        acc[j] = fmaf(xv.z, wv.z, acc[j]);
                        acc[j] = fmaf(xv.w, wv.w, acc[j]);
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (bias) acc[j] += bias[co + j];
            if (relu) acc[j] = max_nan(acc[j], 0.f);
        }
        *reinterpret_cast<float4 *>(y + pix * C + co) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    }
}

// GroupNorm apply (+ optional ReLU, + optional nearest-2x upsampled addend: the FPN top-down step
// laterals[i-1] += interpolate(laterals[i]) of fpn.py:150-154 fused into the lateral's GN)
__global__ void __launch_bounds__(256)
gn_apply_f32_kernel(const float *__restrict__ x, int N, int H, int W, int C, const double *__restrict__ stats,
                    int groups, const float *__restrict__ gamma, const float *__restrict__ beta, float eps,
                    int relu, const float *__restrict__ up, float *__restrict__ y)
{
    const size_t total4 = (size_t)N * H * W * C / 4;
    const int gs = C / groups;
    const double cnt = (double)H * W * gs;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e = i * 4;
        const int c = (int)(e % C);
        const size_t pix = e / C;
        const int n = (int)(pix / ((size_t)H * W));
        float4 v = reinterpret_cast<const float4 *>(x)[i];
        float o[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int g = (c + j) / gs;
            const double s = stats[((size_t)n * groups + g) * 2], q = stats[((size_t)n * groups + g) * 2 + 1];
            const double mean = s / cnt;
            double var = q / cnt - mean * mean;
            var = var < 0 ? 0 : var;
            const float rstd = (float)(1.0 / sqrt(var + (double)eps));
            o[j] = (o[j] - (float)mean) * rstd * gamma[c + j] + beta[c + j];
            if (relu) o[j] = max_nan(o[j], 0.f);
        }
        if (up) {
            const int hw = (int)(pix % ((size_t)H * W));
            const int h = hw / W, w = hw - h * W;
            const int Hu = (H + 1) / 2, Wu = (W + 1) / 2;              // F.interpolate(size=prev_shape, mode='nearest'): src = floor(dst * in / out)
            const float4 u = *reinterpret_cast<const float4 *>(up + (((size_t)n * Hu + (h * Hu) / H) * Wu + (w * Wu) / W) * C + c);
            o[0] += u.x; o[1] += u.y; o[2] += u.z; o[3] += u.w;
        }
        reinterpret_cast<float4 *>(y)[i] = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// max_pool2d(kernel 3, stride 2, padding 1) of resnet.py:497 (nn.MaxPool2d), NHWC
__global__ void __launch_bounds__(256)
maxpool3x3s2_f32_kernel(const float *__restrict__ x, int N, int H, int W, int C, int Ho, int Wo, float *__restrict__ y)
{
    const size_t total4 = (size_t)N * Ho * Wo * C / 4;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t e = i * 4;
        const int c = (int)(e % C);
        const size_t pix = e / C;
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), n = (int)(pix / ((size_t)Wo * Ho));
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
        for (int dh = 0; dh < 3; ++dh)
#pragma unroll
            for (int dw = 0; dw < 3; ++dw) {
                const int ih = oh * 2 - 1 + dh, iw = ow * 2 - 1 + dw;
                if (ih < 0 || ih >= H || iw < 0 || iw >= W) continue;
                const float4 v = *reinterpret_cast<const float4 *>(x + (((size_t)n * H + ih) * W + iw) * C + c);
                m.x = max_nan(v.x, m.x); m.y = max_nan(v.y, m.y); m.z = max_nan(v.z, m.z); m.w = max_nan(v.w, m.w);
            }
        reinterpret_cast<float4 *>(y)[i] = m;
    }
}

// output extent of a convolution: (in + 2 pad - dil (k - 1) - 1) / stride + 1, or 0 when the dilated kernel does not
// fit the padded input (C division truncates toward zero, so a small negative span would otherwise give 1)
int conv_out_extent(int in, int k, int stride, int pad, int dil)
{
    const long long span = (long long)in + 2LL * pad - (long long)dil * (k - 1) - 1;
    return span < 0 ? 0 : (int)(span / stride + 1);
}

int conv_common(const char *name, const float *x, int N, int H, int W, int Cin, const float *w, int Cout, int KH, int KW,
                int stride, int pad, int dil, const float *bias, const float *res, int relu, float *y, double *stats,
                int groups, const float *off, const float *mask, cudaStream_t st)
{
    if (!x || !w || !y) return fail(ORP_EINVAL, "%s: x, w and y must not be NULL", name);
    if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || KH < 1 || KW < 1)
        return fail(ORP_EINVAL, "%s: N, H, W, Cin, Cout, KH and KW must be >= 1", name);
    if (stride < 1 || dil < 1 || pad < 0) return fail(ORP_EINVAL, "%s: stride and dilation must be >= 1, pad >= 0", name);
    if (Cin % 4) return fail(ORP_EINVAL, "%s: Cin must be a multiple of 4 (pad the stem input to 4 channels)", name);
    const int Ho = conv_out_extent(H, KH, stride, pad, dil), Wo = conv_out_extent(W, KW, stride, pad, dil);
    if (Ho < 1 || Wo < 1) return fail(ORP_EINVAL, "%s: the kernel does not fit the padded input (empty output)", name);
    if (stats && (groups < 1 || Cout % groups)) return fail(ORP_EINVAL, "%s: Cout must divide into groups >= 1", name);
    int rc = ensure_device();
    if (rc) return rc;
    ConvP p;
    p.x = x; p.w = w; p.bias = bias; p.res = res; p.off = off; p.mask = mask; p.y = y; p.stats = stats;
    p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout; p.KH = KH; p.KW = KW; p.stride = stride; p.pad = pad; p.dil = dil;
    p.Ho = Ho; p.Wo = Wo;
    p.K = KH * KW * Cin; p.relu = relu; p.groups = groups;
    p.tiles_per_img = ceil_div((long long)p.Ho * p.Wo, BM);
    dim3 grid(N * p.tiles_per_img, ceil_div(Cout, BN));
    if (off) conv_f32_kernel<true><<<grid, 256, 0, st>>>(p);
    else conv_f32_kernel<false><<<grid, 256, 0, st>>>(p);
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace
}  // namespace orp

using namespace orp;

extern "C" int orp_conv2d_f32(const float *x, int N, int H, int W, int Cin, const float *w, int Cout, int KH, int KW,
                              int stride, int pad, const float *bias, const float *residual, int relu, float *y,
                              double *gn_stats, int groups, void *stream)
{
    return conv_common("conv2d_f32", x, N, H, W, Cin, w, Cout, KH, KW, stride, pad, 1, bias, residual, relu, y, gn_stats,
                       groups, nullptr, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" int orp_deform_conv2d_f32(const float *x, int N, int H, int W, int Cin, const float *offset, const float *mask,
                                     const float *w, int Cout, int KH, int KW, int stride, int pad, int dilation,
                                     const float *bias, int relu, float *y, void *stream)
{
    if (!offset) return fail(ORP_EINVAL, "deform_conv2d_f32: offset is NULL");
    return conv_common("deform_conv2d_f32", x, N, H, W, Cin, w, Cout, KH, KW, stride, pad, dilation, bias, nullptr, relu, y,
                       nullptr, 0, offset, mask, static_cast<cudaStream_t>(stream));
}

/* see include/orp_b200_group.h */
extern "C" int orp_group_conv2d_f32(const float *x, int N, int H, int W, int width, int groups, const float *w, int stride,
                                    const float *bias, int relu, float *y, void *stream)
{
    if (!x || !w || !y) return fail(ORP_EINVAL, "group_conv2d_f32: x, w and y must not be NULL");
    if (N < 1 || H < 1 || W < 1 || width < 1 || stride < 1) return fail(ORP_EINVAL, "group_conv2d_f32: N, H, W, width and stride must be >= 1");
    if (groups < 1 || width % groups || (width / groups) % 4)
        return fail(ORP_EINVAL, "group_conv2d_f32: width must divide into groups of a multiple of 4 channels");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = conv_out_extent(H, 3, stride, 1, 1), Wo = conv_out_extent(W, 3, stride, 1, 1);
    const size_t total = (size_t)N * Ho * Wo * (width / 4);
    int grid = (int)((total + 255) / 256);
    if (grid > kNumSMs * 16) grid = kNumSMs * 16;
    group_conv3x3_f32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, N, H, W, width, width / groups, w, stride, Ho, Wo,
                                                                                  bias, relu, y);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_gn_apply_f32(const float *x, int N, int H, int W, int C, const double *stats, int groups,
                                const float *gamma, const float *beta, float eps, int relu, const float *up_src, float *y,
                                void *stream)
{
    if (!x || !y || !stats || !gamma || !beta) return fail(ORP_EINVAL, "gn_apply_f32: x, stats, gamma, beta and y must not be NULL");
    if (N < 1 || H < 1 || W < 1 || C < 1) return fail(ORP_EINVAL, "gn_apply_f32: N, H, W and C must be >= 1");
    if (C % 4) return fail(ORP_EINVAL, "gn_apply_f32: C must be a multiple of 4");
    if (groups < 1 || C % groups) return fail(ORP_EINVAL, "gn_apply_f32: C must divide into groups >= 1");
    int rc = ensure_device();
    if (rc) return rc;
    const size_t total4 = (size_t)N * H * W * C / 4;
    int grid = (int)((total4 + 255) / 256);
    if (grid > kNumSMs * 16) grid = kNumSMs * 16;
    gn_apply_f32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, N, H, W, C, stats, groups, gamma, beta, eps,
                                                                             relu, up_src, y);
    ORP_LAUNCHED();
    return ORP_OK;
}

extern "C" int orp_maxpool3x3s2_f32(const float *x, int N, int H, int W, int C, float *y, void *stream)
{
    if (!x || !y) return fail(ORP_EINVAL, "maxpool3x3s2_f32: x and y must not be NULL");
    if (N < 1 || H < 1 || W < 1 || C < 1) return fail(ORP_EINVAL, "maxpool3x3s2_f32: N, H, W and C must be >= 1");
    if (C % 4) return fail(ORP_EINVAL, "maxpool3x3s2_f32: C must be a multiple of 4");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    const size_t total4 = (size_t)N * Ho * Wo * C / 4;
    int grid = (int)((total4 + 255) / 256);
    if (grid > kNumSMs * 16) grid = kNumSMs * 16;
    maxpool3x3s2_f32_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, N, H, W, C, Ho, Wo, y);
    ORP_LAUNCHED();
    return ORP_OK;
}

/* see include/orp_b200_hrnet.h */
extern "C" int orp_hr_fuse_f32(const float *base, int N, int H, int W, int C, int nsrc, const float *const *src, float *y, void *stream)
{
    return orp::hr_fuse<orp::ActF32>(base, N, H, W, C, nsrc, reinterpret_cast<const void *const *>(src), y, stream, "hr_fuse_f32");
}

extern "C" int orp_hrfpn_reduce_f32(int nparts, const float *const *part, int N, int H, int W, int C, float *y, void *stream)
{
    return orp::hrfpn_reduce<orp::ActF32>(nparts, part, N, H, W, C, y, stream, "hrfpn_reduce_f32");
}

extern "C" int orp_hrfpn_pool_f32(const float *x, int N, int H, int W, int C, int max_pool, float *const *out, void *stream)
{
    return orp::hrfpn_pool<orp::ActF32>(x, N, H, W, C, max_pool, reinterpret_cast<void *const *>(out), stream, "hrfpn_pool_f32");
}
