// act.cuh - element access of the tensor-core engines' two activation formats, so that a memory-bound kernel is written
// once for both: bf16 [.., C] and the f16x3 "split" format fp16 [.., 2, C] (per token C hi values, then C lo values,
// x = hi + lo).  The arithmetic in between is fp32 either way.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace orp {

// token-wise element access: `tok` = token (pixel) index, C = channels per token
template <bool SPLIT> struct Act;
template <> struct Act<false> {
    typedef __nv_bfloat16 T;
    static __device__ __forceinline__ float ld(const T *b, long long tok, int C, int c) { return __bfloat162float(b[tok * C + c]); }
    static __device__ __forceinline__ void st(T *b, long long tok, int C, int c, float v) { b[tok * C + c] = __float2bfloat16_rn(v); }
    static constexpr int planes = 1;
    // 8 consecutive channels (c % 8 == 0) of one token
    static __device__ __forceinline__ void ld8(const T *b, long long tok, int C, int c, float (&o)[8])
    {
        const uint4 u = *reinterpret_cast<const uint4 *>(b + tok * C + c);
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&w[k]));
            o[2 * k] = f.x; o[2 * k + 1] = f.y;
        }
    }
    // 8 values to p (16-byte aligned); `lo` is the split format's offset of the lo half, unused here
    static __device__ __forceinline__ void st8(T *p, long long /*lo*/, const float (&v)[8])
    {
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            __nv_bfloat162 q = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
            w[k] = *reinterpret_cast<uint32_t *>(&q);
        }
        *reinterpret_cast<uint4 *>(p) = make_uint4(w[0], w[1], w[2], w[3]);
    }
    static __device__ __forceinline__ void st8(T *b, long long tok, int C, int c, const float (&v)[8]) { st8(b + tok * C + c, 0, v); }
};
template <> struct Act<true> {
    typedef __half T;
    static __device__ __forceinline__ float ld(const T *b, long long tok, int C, int c)
    {
        const T *p = b + tok * 2 * C + c;
        return __half2float(p[0]) + __half2float(p[C]);
    }
    // values beyond the fp16 range saturate (the convolutions count such events)
    static __device__ __forceinline__ void st(T *b, long long tok, int C, int c, float v)
    {
        const float a = fminf(fmaxf(v, -65504.f), 65504.f);
        const __half h = __float2half_rn(a);
        T *p = b + tok * 2 * C + c;
        p[0] = h;
        p[C] = __float2half_rn(a - __half2float(h));
    }
    static constexpr int planes = 2;
    static __device__ __forceinline__ void ld8(const T *b, long long tok, int C, int c, float (&o)[8])
    {
        const T *p = b + tok * 2 * C + c;
        const uint4 uh = *reinterpret_cast<const uint4 *>(p), ul = *reinterpret_cast<const uint4 *>(p + C);
        const uint32_t wh[4] = {uh.x, uh.y, uh.z, uh.w}, wl[4] = {ul.x, ul.y, ul.z, ul.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 fh = __half22float2(*reinterpret_cast<const __half2 *>(&wh[k]));
            const float2 fl = __half22float2(*reinterpret_cast<const __half2 *>(&wl[k]));
            o[2 * k] = fh.x + fl.x; o[2 * k + 1] = fh.y + fl.y;      // exact: the pair has at most 22 significant bits
        }
    }
    // 8 values: hi halves to p, lo halves to p + lo (16-byte aligned)
    static __device__ __forceinline__ void st8(T *p, long long lo, const float (&v)[8])
    {
        uint32_t wh[4], wl[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float a = fminf(fmaxf(v[2 * k], -65504.f), 65504.f), d = fminf(fmaxf(v[2 * k + 1], -65504.f), 65504.f);
            const __half2 h2 = __floats2half2_rn(a, d);
            const float2 hf = __half22float2(h2);
            const __half2 l2 = __floats2half2_rn(a - hf.x, d - hf.y);
            wh[k] = *reinterpret_cast<const uint32_t *>(&h2);
            wl[k] = *reinterpret_cast<const uint32_t *>(&l2);
        }
        *reinterpret_cast<uint4 *>(p) = make_uint4(wh[0], wh[1], wh[2], wh[3]);
        *reinterpret_cast<uint4 *>(p + lo) = make_uint4(wl[0], wl[1], wl[2], wl[3]);
    }
    static __device__ __forceinline__ void st8(T *b, long long tok, int C, int c, const float (&v)[8]) { st8(b + tok * 2 * C + c, C, v); }
};

}  // namespace orp
