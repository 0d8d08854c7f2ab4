// minarearect.cu - 9-point sets -> minimum-area rectangles on sm_90a (SURVEY.md section 8 row a8).
//
// Replaces minareabbox_cuda (mmdet/ops/minarearect/src/minarearect_kernel.cu:470-505), which runs one
// thread per set on the legacy stream, then copies the result to the host, loops over it and uploads it
// again.  Here: one thread per set on the caller's stream, inputs staged through shared memory with
// coalesced 128-bit loads (72 B in / 32 B out per set = 104 B algorithmic, HBM-bound), the result stays
// on the device and the `* stride + centre` affine of orientedreppoints_head.py:748-749 can be fused in.
//
// Arithmetic: the reference's mixed precision, operation for operation, with the round-to-nearest
// intrinsics so nothing is contracted (see oracle/oracle_minarearect.c for the statement of the
// three deliberate differences: double-evaluated cos, no FMA, bounded gift-wrapping loops).
#include "common.cuh"
#include "minrect.cuh"

namespace orp {

namespace {

using namespace orp::mr;

constexpr int kThreads = 128;

__global__ void __launch_bounds__(kThreads)
minarearect_kernel(const float *__restrict__ pts, int n, float *__restrict__ out,
                   int32_t *__restrict__ hull_map, float scale, const float *__restrict__ center)
{
    __shared__ float s_in[kThreads * 18];
    __shared__ float s_out[kThreads * 8];
    const int base = blockIdx.x * kThreads;
    const int cnt = min(kThreads, n - base);
    // coalesced staging: the block's rows are one contiguous span of cnt*18 floats
    {
        const float *src = pts + (size_t)base * 18;
        const int total = cnt * 18;
        const bool al16 = ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
        if (al16) {
            const int nv = total >> 2;
            const float4 *s4 = reinterpret_cast<const float4 *>(src);
            float4 *d4 = reinterpret_cast<float4 *>(s_in);
            for (int t = threadIdx.x; t < nv; t += kThreads) d4[t] = s4[t];
            for (int t = (nv << 2) + threadIdx.x; t < total; t += kThreads) s_in[t] = src[t];
        } else {
            for (int t = threadIdx.x; t < total; t += kThreads) s_in[t] = src[t];
        }
    }
    __syncthreads();
    if (threadIdx.x < cnt) {
        float in[18], o[8];
        int32_t map[9];
#pragma unroll
        for (int k = 0; k < 18; ++k) in[k] = s_in[threadIdx.x * 18 + k];   // stride 18: conflict-free (gcd(18,32)=2 -> 2-way)
        minrect_one(in, o, hull_map ? map : nullptr);
        if (center) {
            const float cxv = center[(size_t)(base + threadIdx.x) * 2], cyv = center[(size_t)(base + threadIdx.x) * 2 + 1];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                o[2 * c] = __fadd_rn(__fmul_rn(o[2 * c], scale), cxv);
                o[2 * c + 1] = __fadd_rn(__fmul_rn(o[2 * c + 1], scale), cyv);
            }
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) s_out[threadIdx.x * 8 + k] = o[k];
        if (hull_map)
#pragma unroll
            for (int k = 0; k < 9; ++k) hull_map[(size_t)(base + threadIdx.x) * 9 + k] = map[k];
    }
    __syncthreads();
    {
        float *dst = out + (size_t)base * 8;   // 32 B per row: always 16 B aligned if `out` is
        const int total = cnt * 8;
        if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            float4 *d4 = reinterpret_cast<float4 *>(dst);
            const float4 *s4 = reinterpret_cast<const float4 *>(s_out);
            for (int t = threadIdx.x; t < (total >> 2); t += kThreads) d4[t] = s4[t];
        } else {
            for (int t = threadIdx.x; t < total; t += kThreads) dst[t] = s_out[t];
        }
    }
}

}  // namespace
}  // namespace orp

extern "C" int orp_minarearect(const float *pts, int n, float *out, int32_t *hull_map, float scale,
                               const float *center, void *stream)
{
    using namespace orp;
    if (n < 0 || (n > 0 && (!pts || !out))) return fail(ORP_EINVAL, "orp_minarearect: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    if (n == 0) return ORP_OK;
    minarearect_kernel<<<ceil_div(n, kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        pts, n, out, hull_map, scale, center);
    ORP_LAUNCHED();
    return ORP_OK;
}
