// hrnet.cuh - the memory-bound layers of HRNet and HRFPN (include/orp_b200_hrnet.h), written once over the activation
// format: Act<false> (bf16), Act<true> (f16x3 split) from act.cuh, and ActF32 (fp32, the CUDA-core engine) below.  hrnet.cu
// instantiates the tensor-core formats, dense_f32.cu the fp32 one.  Every kernel moves whole 16-byte channel vectors
// (8 channels per item) and computes in fp32; split-format stores saturate and are counted.
#pragma once
#include <math.h>

#include "act.cuh"
#include "common.cuh"

namespace orp {

// fp32 NHWC [.., C], the same interface as Act<>
struct ActF32 {
    typedef float T;
    static constexpr int planes = 1;
    static __device__ __forceinline__ void ld8(const T *b, long long tok, int C, int c, float (&o)[8])
    {
        const float4 a = *reinterpret_cast<const float4 *>(b + tok * C + c), d = *reinterpret_cast<const float4 *>(b + tok * C + c + 4);
        o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = d.x; o[5] = d.y; o[6] = d.z; o[7] = d.w;
    }
    static __device__ __forceinline__ void st8(T *b, long long tok, int C, int c, const float (&v)[8])
    {
        *reinterpret_cast<float4 *>(b + tok * C + c) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4 *>(b + tok * C + c + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
};

// dense_tc.cu: the device address of the f16x3 saturation counter that orp_f16x3_overflow_count reads
unsigned int *f16x3_overflow_counter();

namespace {

// 8 values of one token; in the split format a value beyond the fp16 range saturates and the vector counts once
template <class A>
__device__ __forceinline__ void store8(typename A::T *b, long long tok, int C, int c, const float (&v)[8], unsigned int *ovf)
{
    if constexpr (A::planes == 2) {
        float m = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) m = fmaxf(m, fabsf(v[j]));
        if (m > 65504.f) atomicAdd(ovf, 1u);
    }
    A::st8(b, tok, C, c, v);
}

template <typename T> struct HrFuseP {
    const T *base;
    const T *src[3];
    T *y;
    int N, H, W, C, nsrc;
    unsigned int *ovf;
};

// y = relu(base + sum_k nearest_up(src[k-1], 2^k)): one item = (pixel, 8 channels)
template <class A>
__global__ void __launch_bounds__(256) hr_fuse_kernel(const __grid_constant__ HrFuseP<typename A::T> P)
{
    const int c8 = P.C / 8;
    const size_t total = (size_t)P.N * P.H * P.W * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c8) * 8;
        const size_t pix = i / c8;
        const int x = (int)(pix % P.W), y = (int)((pix / P.W) % P.H);
        const size_t n = pix / ((size_t)P.W * P.H);
        float v[8];
        A::ld8(P.base, (long long)pix, P.C, c, v);
#pragma unroll
        for (int k = 1; k <= 3; ++k) {
            if (k > P.nsrc) break;
            const int hk = P.H >> k, wk = P.W >> k;
            float u[8];
            A::ld8(P.src[k - 1], (long long)((n * hk + (y >> k)) * wk + (x >> k)), P.C, c, u);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += u[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = v[j] < 0.f ? 0.f : v[j];       // nn.ReLU: NaN stays NaN
        store8<A>(P.y, (long long)pix, P.C, c, v, P.ovf);
    }
}

template <typename T> struct HrReduceP {
    const float *part[4];
    T *y;
    int nparts, N, H, W, C;
    unsigned int *ovf;
};

// y = sum_i bilinear_up(part[i], 2^i) (align_corners=False): one item = (pixel, 8 channels)
template <class A>
__global__ void __launch_bounds__(256) hrfpn_reduce_kernel(const __grid_constant__ HrReduceP<typename A::T> P)
{
    const int c8 = P.C / 8;
    const size_t total = (size_t)P.N * P.H * P.W * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c8) * 8;
        const size_t pix = i / c8;
        const int x = (int)(pix % P.W), y = (int)((pix / P.W) % P.H);
        const size_t n = pix / ((size_t)P.W * P.H);
        float v[8];
        ActF32::ld8(P.part[0], (long long)pix, P.C, c, v);
#pragma unroll
        for (int k = 1; k < 4; ++k) {
            if (k >= P.nparts) break;
            const int hk = P.H >> k, wk = P.W >> k;
            const float inv = 1.f / (float)(1 << k);                              // exact: a power of two
            // area_pixel_compute_source_index (align_corners=False): src = (dst + 0.5) / scale - 0.5, clamped at 0
            const float sy = fmaxf(((float)y + 0.5f) * inv - 0.5f, 0.f), sx = fmaxf(((float)x + 0.5f) * inv - 0.5f, 0.f);
            const int y0 = (int)sy, x0 = (int)sx;
            const int y1 = min(y0 + 1, hk - 1), x1 = min(x0 + 1, wk - 1);
            const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.f - ly, hx = 1.f - lx;
            const float *p = P.part[k];
            float a[8], b[8], d[8], e[8];
            ActF32::ld8(p, (long long)((n * hk + y0) * wk + x0), P.C, c, a);
            ActF32::ld8(p, (long long)((n * hk + y0) * wk + x1), P.C, c, b);
            ActF32::ld8(p, (long long)((n * hk + y1) * wk + x0), P.C, c, d);
            ActF32::ld8(p, (long long)((n * hk + y1) * wk + x1), P.C, c, e);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += hy * (hx * a[j] + lx * b[j]) + ly * (hx * d[j] + lx * e[j]);
        }
        store8<A>(P.y, (long long)pix, P.C, c, v, P.ovf);
    }
}

template <typename T> struct HrPoolP {
    const T *x;
    T *out[4];
    int N, H, W, C, maxp;
    unsigned int *ovf;
};

__device__ __forceinline__ float pool_op(bool maxp, float a, float b)
{
    return maxp ? ((a > b || a != a) ? a : b) : a + b;                      // max_pool2d keeps a NaN
}

// The four pooled levels from one read of x.  A warp covers one 16 x 16 cell for 2 channel vectors: lane = (16 x 16 cell's
// 4 x 4 window in Morton order: bit 0 / 2 = x, bit 1 / 3 = y) + 16 * (vector).  Each lane reduces its 2 x 2 and 4 x 4
// windows from memory; shuffles over lane bits 0-1 give the 8 x 8 windows and bits 2-3 the 16 x 16 one.  A window is
// written only when it lies inside the map (floor semantics); lanes outside still take part in the shuffles.
template <class A>
__global__ void __launch_bounds__(256) hrfpn_pool_kernel(const __grid_constant__ HrPoolP<typename A::T> P)
{
    const int lane = threadIdx.x & 31, sub = lane & 15;
    const int c8 = P.C / 8, cpairs = (c8 + 1) / 2;
    const int Hc = (P.H + 15) / 16, Wc = (P.W + 15) / 16;
    const long long ngroups = (long long)P.N * Hc * Wc * cpairs;
    const long long warps = (long long)gridDim.x * (blockDim.x / 32);
    const bool maxp = P.maxp != 0;
    const float ident = maxp ? -INFINITY : 0.f;
    const int sx = (sub & 1) | ((sub >> 1) & 2), sy = ((sub >> 1) & 1) | ((sub >> 2) & 2);
    for (long long g = blockIdx.x * (long long)(blockDim.x / 32) + (threadIdx.x >> 5); g < ngroups; g += warps) {
        const int cp = (int)(g % cpairs);
        const long long cell = g / cpairs;
        const int cx = (int)(cell % Wc), cy = (int)((cell / Wc) % Hc);
        const long long n = cell / ((long long)Wc * Hc);
        const int chunk = 2 * cp + (lane >> 4), c = chunk * 8;
        const bool active = chunk < c8;
        const int y0 = cy * 16 + sy * 4, x0 = cx * 16 + sx * 4;
        float a4[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) a4[j] = ident;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int py = y0 + 2 * (q >> 1), px = x0 + 2 * (q & 1);
            if (!active || py + 2 > P.H || px + 2 > P.W) continue;          // then the 4 x 4 window is partial too
            float a2[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) a2[j] = ident;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                float v[8];
                A::ld8(P.x, (n * P.H + py + (t >> 1)) * P.W + px + (t & 1), P.C, c, v);
#pragma unroll
                for (int j = 0; j < 8; ++j) a2[j] = pool_op(maxp, a2[j], v[j]);
            }
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { o[j] = maxp ? a2[j] : a2[j] * 0.25f; a4[j] = pool_op(maxp, a4[j], a2[j]); }
            store8<A>(P.out[0], (n * (P.H >> 1) + (py >> 1)) * (P.W >> 1) + (px >> 1), P.C, c, o, P.ovf);
        }
        if (active && y0 + 4 <= P.H && x0 + 4 <= P.W) {
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = maxp ? a4[j] : a4[j] * 0.0625f;
            store8<A>(P.out[1], (n * (P.H >> 2) + (y0 >> 2)) * (P.W >> 2) + (x0 >> 2), P.C, c, o, P.ovf);
        }
        float a8[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            a8[j] = pool_op(maxp, a4[j], __shfl_xor_sync(0xffffffffu, a4[j], 1));
            a8[j] = pool_op(maxp, a8[j], __shfl_xor_sync(0xffffffffu, a8[j], 2));
        }
        const int y8 = y0 & ~7, x8 = x0 & ~7;
        if (active && (sub & 3) == 0 && y8 + 8 <= P.H && x8 + 8 <= P.W) {
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = maxp ? a8[j] : a8[j] * (1.f / 64.f);
            store8<A>(P.out[2], (n * (P.H >> 3) + (y8 >> 3)) * (P.W >> 3) + (x8 >> 3), P.C, c, o, P.ovf);
        }
        float a16[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            a16[j] = pool_op(maxp, a8[j], __shfl_xor_sync(0xffffffffu, a8[j], 4));
            a16[j] = pool_op(maxp, a16[j], __shfl_xor_sync(0xffffffffu, a16[j], 8));
        }
        if (active && sub == 0 && cy * 16 + 16 <= P.H && cx * 16 + 16 <= P.W) {
            float o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o[j] = maxp ? a16[j] : a16[j] * (1.f / 256.f);
            store8<A>(P.out[3], (n * (P.H >> 4) + cy) * (P.W >> 4) + cx, P.C, c, o, P.ovf);
        }
    }
}

inline bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

inline bool bad_dims(int N, int H, int W, int C) { return N < 1 || H < 1 || W < 1 || C < 8 || C % 8; }

inline int overflow_ptr(bool split, unsigned int *&ovf, const char *name)
{
    ovf = nullptr;
    if (split && !(ovf = f16x3_overflow_counter())) return fail(ORP_ECUDA, "%s: no overflow counter", name);
    return ORP_OK;
}

template <class A>
int hr_fuse(const void *base, int N, int H, int W, int C, int nsrc, const void *const *src, void *y, void *stream, const char *name)
{
    typedef typename A::T T;
    if (!base || !y || !src || bad_dims(N, H, W, C) || nsrc < 1 || nsrc > 3)
        return fail(ORP_EINVAL, "%s: needs base, y, 1..3 sources, N, H, W >= 1 and C a multiple of 8", name);
    if (H % (1 << nsrc) || W % (1 << nsrc)) return fail(ORP_EINVAL, "%s: H and W must be multiples of 2^nsrc", name);
    HrFuseP<T> P{};
    P.base = static_cast<const T *>(base);
    P.y = static_cast<T *>(y);
    for (int k = 0; k < nsrc; ++k) {
        if (!src[k] || !aligned16(src[k]) || src[k] == y) return fail(ORP_EINVAL, "%s: every source must be a 16-byte aligned pointer other than y", name);
        P.src[k] = static_cast<const T *>(src[k]);
    }
    if (!aligned16(base) || !aligned16(y) || base == y) return fail(ORP_EINVAL, "%s: base and y must be distinct 16-byte aligned pointers", name);
    P.N = N; P.H = H; P.W = W; P.C = C; P.nsrc = nsrc;
    int rc = overflow_ptr(A::planes == 2, P.ovf, name);
    if (rc || (rc = ensure_device())) return rc;
    hr_fuse_kernel<A><<<grid_for((size_t)N * H * W * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

template <class A>
int hrfpn_reduce(int nparts, const float *const *part, int N, int H, int W, int C, void *y, void *stream, const char *name)
{
    typedef typename A::T T;
    if (!part || !y || bad_dims(N, H, W, C) || nparts < 1 || nparts > 4)
        return fail(ORP_EINVAL, "%s: needs 1..4 parts, y, N, H, W >= 1 and C a multiple of 8", name);
    const int m = 1 << (nparts - 1);
    if (H % m || W % m) return fail(ORP_EINVAL, "%s: H and W must be multiples of 2^(nparts-1)", name);
    HrReduceP<T> P{};
    for (int k = 0; k < nparts; ++k) {
        if (!part[k] || !aligned16(part[k]) || (const void *)part[k] == y)
            return fail(ORP_EINVAL, "%s: every part must be a 16-byte aligned pointer other than y", name);
        P.part[k] = part[k];
    }
    if (!aligned16(y)) return fail(ORP_EINVAL, "%s: y must be 16-byte aligned", name);
    P.y = static_cast<T *>(y);
    P.nparts = nparts; P.N = N; P.H = H; P.W = W; P.C = C;
    int rc = overflow_ptr(A::planes == 2, P.ovf, name);
    if (rc || (rc = ensure_device())) return rc;
    hrfpn_reduce_kernel<A><<<grid_for((size_t)N * H * W * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

template <class A>
int hrfpn_pool(const void *x, int N, int H, int W, int C, int max_pool, void *const *out, void *stream, const char *name)
{
    typedef typename A::T T;
    if (!x || !out || bad_dims(N, H, W, C) || (max_pool != 0 && max_pool != 1))
        return fail(ORP_EINVAL, "%s: needs x, out, N, H, W >= 1, C a multiple of 8 and max_pool 0 or 1", name);
    if (!aligned16(x)) return fail(ORP_EINVAL, "%s: x must be 16-byte aligned", name);
    HrPoolP<T> P{};
    P.x = static_cast<const T *>(x);
    for (int l = 0; l < 4; ++l) {
        const bool used = (H >> (l + 1)) > 0 && (W >> (l + 1)) > 0;
        if (used && (!out[l] || !aligned16(out[l]) || out[l] == x))
            return fail(ORP_EINVAL, "%s: every level that is not empty needs a 16-byte aligned output other than x", name);
        P.out[l] = static_cast<T *>(out[l]);
    }
    P.N = N; P.H = H; P.W = W; P.C = C; P.maxp = max_pool;
    int rc = overflow_ptr(A::planes == 2, P.ovf, name);
    if (rc || (rc = ensure_device())) return rc;
    const size_t groups = (size_t)N * ((H + 15) / 16) * ((W + 15) / 16) * ((C / 8 + 1) / 2);
    hrfpn_pool_kernel<A><<<grid_for(groups * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace
}  // namespace orp
