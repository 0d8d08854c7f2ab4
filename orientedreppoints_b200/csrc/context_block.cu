// context_block.cu - the global context block (GCB) of ResNet / ResNeXt bottlenecks (include/orp_b200_context.h,
// mmdet/ops/context_block.py), in the three activation formats of the engines.
//
// Pool: one CTA per (chunk of pixels, image).  A CTA holds `slots` pixel slots of warps_per_slot warps; lane l of a slot's
// warp w owns the 8 channels of vector w * 32 + l, so a slot covers a whole pixel (C <= 2048) and reads it as contiguous
// 16-byte vectors.  Each slot takes kPix pixels per pass: the logits (per-lane 8-product partials, a butterfly over the warp
// and, for a slot of several warps, a fixed-order sum through shared memory), then an fp32 online softmax update of its
// running max, sum and exp-weighted channel sums.  At the end the slots are combined in order and the chunk's partials
// written.  'avg' is the same walk with every logit 0: max 0, sum = pixel count, plain channel sums.  x is read once.
// Transform: one CTA per (image, fusion): the chunks combined in order, then 1x1 -> LayerNorm -> ReLU -> 1x1 (-> sigmoid),
// each dot product a warp's fixed-order butterfly.  Fuse: one item = (pixel, 8 channels), as the HRNet fuse adds.
// No float atomics: every sum has one order, so the results are bitwise reproducible.
#include <math.h>

#include "hrnet.cuh"
#include "../../include/orp_b200_context.h"

namespace orp {
namespace {

constexpr int kPix = 4;                 // pixels per slot and pass
constexpr int kPoolThreads = 256;       // eight warps
constexpr int kTargetCtas = 4 * kNumSMs;
constexpr int kMaxC = 2048;             // eight warps of 32 lanes x 8 channels: one pixel per CTA pass
constexpr int kMaxChunks = 1024;
constexpr int kTransformThreads = 512;

__device__ __forceinline__ float warp_sum(float a)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);     // every lane ends with the same bits
    return a;
}

struct PoolP {
    const void *x;
    const float *w;                     // conv_mask weight [C], NULL: 'avg'
    float *ws;
    int N, HW, C, chunks, L, slots, wps;
};

template <class A>
__global__ void __launch_bounds__(kPoolThreads) context_pool_kernel(const __grid_constant__ PoolP P)
{
    __shared__ float red[2][8][kPix];   // per warp and pass: its lanes' logit sum
    __shared__ float slot_m[8], slot_s[8];
    __shared__ float sctx[kMaxC];       // slots * C <= 2048: the slots' rescaled channel sums
    const typename A::T *x = static_cast<const typename A::T *>(P.x);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int slot = warp / P.wps, wis = warp % P.wps;
    const int c = (wis * 32 + lane) * 8;
    const bool act = c < P.C;
    const bool att = P.w != nullptr;
    const int n = blockIdx.y, chunk = blockIdx.x;
    const long long p0 = (long long)chunk * P.L;
    const long long p1 = min(p0 + P.L, (long long)P.HW);
    const long long img = (long long)n * P.HW;
    float wv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) wv[j] = (att && act) ? P.w[c + j] : 0.f;
    float m = -INFINITY, s = 0.f, acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    const int step = P.slots * kPix;
    int buf = 0;
    for (long long base = p0; base < p1; base += step) {            // the same trip count in every thread of the CTA
        float xv[kPix][8], l[kPix];
#pragma unroll
        for (int u = 0; u < kPix; ++u) {
            const long long pix = base + slot * kPix + u;
            if (act && pix < p1) {
                A::ld8(x, img + pix, P.C, c, xv[u]);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) xv[u][j] = 0.f;
            }
        }
        if (att) {
#pragma unroll
            for (int u = 0; u < kPix; ++u) {
                float d = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) d = fmaf(wv[j], xv[u][j], d);
                l[u] = warp_sum(d);
            }
            if (P.wps > 1) {
                if (lane == 0) {
#pragma unroll
                    for (int u = 0; u < kPix; ++u) red[buf][warp][u] = l[u];
                }
                __syncthreads();
#pragma unroll
                for (int u = 0; u < kPix; ++u) {
                    float d = 0.f;
                    for (int k = 0; k < P.wps; ++k) d += red[buf][slot * P.wps + k][u];
                    l[u] = d;
                }
                buf ^= 1;                                         // the next pass writes the other buffer: one barrier per pass
            }
        } else {
#pragma unroll
            for (int u = 0; u < kPix; ++u) l[u] = 0.f;
        }
        float lm = -INFINITY;
#pragma unroll
        for (int u = 0; u < kPix; ++u) {
            if (base + slot * kPix + u >= p1) l[u] = -INFINITY;
            lm = fmaxf(lm, l[u]);
        }
        const float mn = fmaxf(m, lm);
        if (mn != -INFINITY) {                                    // uniform over the slot; false only for a slot past the chunk
            const float sc = expf(m - mn);
            s *= sc;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[j] *= sc;
#pragma unroll
            for (int u = 0; u < kPix; ++u) {
                const float p = expf(l[u] - mn);
                s += p;
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[j] = fmaf(p, xv[u][j], acc[j]);
            }
            m = mn;
        }
    }
    if (threadIdx.x == slot * P.wps * 32) { slot_m[slot] = m; slot_s[slot] = s; }
    __syncthreads();
    float M = -INFINITY;
    for (int k = 0; k < P.slots; ++k) M = fmaxf(M, slot_m[k]);
    const float sc = m == -INFINITY ? 0.f : expf(m - M);
    if (act) {
#pragma unroll
        for (int j = 0; j < 8; ++j) sctx[slot * P.C + c + j] = acc[j] * sc;
    }
    __syncthreads();
    const long long rec = (long long)n * P.chunks + chunk;
    float *out = P.ws + rec * P.C;
    for (int cc = threadIdx.x; cc < P.C; cc += blockDim.x) {
        float a = 0.f;
        for (int k = 0; k < P.slots; ++k) a += sctx[k * P.C + cc];
        out[cc] = a;
    }
    if (threadIdx.x == 0) {
        float S = 0.f;
        for (int k = 0; k < P.slots; ++k) S += slot_m[k] == -INFINITY ? 0.f : slot_s[k] * expf(slot_m[k] - M);
        float *ms = P.ws + (long long)P.N * P.chunks * P.C + 2 * rec;
        ms[0] = M;
        ms[1] = S;
    }
}

struct TransformP {
    const float *ws;
    int N, chunks, C, P;
    orp_context_mlp mlp[2];
    float *out[2];
    int sigmoid[2];
};

__global__ void __launch_bounds__(kTransformThreads) context_transform_kernel(const __grid_constant__ TransformP T)
{
    __shared__ float sscale[kMaxChunks];
    __shared__ float sctx[kMaxC];
    __shared__ float sh[kMaxC];
    __shared__ float sred[3];
    const int n = blockIdx.x, f = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const orp_context_mlp *mp = f ? &T.mlp[1] : &T.mlp[0];
    const float *ms = T.ws + (long long)T.N * T.chunks * T.C + 2LL * n * T.chunks;
    // 1. the chunks' common max M, their weights exp(m_j - M) and the total weight S
    if (warp == 0) {
        float M = -INFINITY;
        for (int j = lane; j < T.chunks; j += 32) M = fmaxf(M, ms[2 * j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));
        float S = 0.f;
        for (int j = lane; j < T.chunks; j += 32) {
            const float e = ms[2 * j] == -INFINITY ? 0.f : expf(ms[2 * j] - M);
            sscale[j] = e;
            S += e * ms[2 * j + 1];
        }
        S = warp_sum(S);
        if (lane == 0) sred[0] = 1.f / S;
    }
    __syncthreads();
    const float inv = sred[0];
    const float *rec = T.ws + (long long)n * T.chunks * T.C;
    for (int c = threadIdx.x; c < T.C; c += blockDim.x) {
        float a = 0.f;
        for (int j = 0; j < T.chunks; ++j) a = fmaf(sscale[j], rec[(long long)j * T.C + c], a);
        sctx[c] = a * inv;
    }
    __syncthreads();
    // 2. h = w1 ctx + b1 (a warp per row)
    for (int o = warp; o < T.P; o += nwarps) {
        const float4 *row = reinterpret_cast<const float4 *>(mp->w1 + (long long)o * T.C);
        float a = 0.f;
        for (int q = lane; q < T.C / 4; q += 32) {
            const float4 w = row[q];
            a = fmaf(w.x, sctx[4 * q], a);
            a = fmaf(w.y, sctx[4 * q + 1], a);
            a = fmaf(w.z, sctx[4 * q + 2], a);
            a = fmaf(w.w, sctx[4 * q + 3], a);
        }
        a = warp_sum(a);
        if (lane == 0) sh[o] = a + mp->b1[o];
    }
    __syncthreads();
    // 3. LayerNorm([P, 1, 1]) over the P values (biased variance, eps 1e-5), ReLU
    if (warp == 0) {
        float a = 0.f;
        for (int o = lane; o < T.P; o += 32) a += sh[o];
        const float mean = warp_sum(a) / (float)T.P;
        float v = 0.f;
        for (int o = lane; o < T.P; o += 32) v = fmaf(sh[o] - mean, sh[o] - mean, v);
        const float var = warp_sum(v) / (float)T.P;
        if (lane == 0) { sred[1] = mean; sred[2] = 1.f / sqrtf(var + 1e-5f); }
    }
    __syncthreads();
    const float mean = sred[1], rstd = sred[2];
    for (int o = threadIdx.x; o < T.P; o += blockDim.x) {
        const float v = (sh[o] - mean) * rstd * mp->ln_w[o] + mp->ln_b[o];
        sh[o] = v < 0.f ? 0.f : v;                                    // nn.ReLU: NaN stays NaN
    }
    __syncthreads();
    // 4. t = w2 h + b2 (a warp per output channel), sigmoid for channel_mul
    float *out = (f ? T.out[1] : T.out[0]) + (long long)n * T.C;
    const bool sig = f ? T.sigmoid[1] : T.sigmoid[0];
    for (int c = warp; c < T.C; c += nwarps) {
        const float *row = mp->w2 + (long long)c * T.P;
        float a = 0.f;
        for (int o = lane; o < T.P; o += 32) a = fmaf(row[o], sh[o], a);
        a = warp_sum(a);
        if (lane == 0) {
            const float v = a + mp->b2[c];
            out[c] = sig ? 1.f / (1.f + expf(-v)) : v;
        }
    }
}

// y = relu(x * mul[n] + add[n] + identity): one item = (pixel, 8 channels)
template <class A>
__global__ void __launch_bounds__(256) context_fuse_kernel(const typename A::T *x, const typename A::T *idt, int N, int HW, int C,
                                                           const float *mul, const float *add, typename A::T *y, unsigned int *ovf)
{
    const int c8 = C / 8;
    const size_t total = (size_t)N * HW * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c8) * 8;
        const size_t pix = i / c8, n = pix / HW;
        float v[8], r[8], t[8];
        A::ld8(x, (long long)pix, C, c, v);
        A::ld8(idt, (long long)pix, C, c, r);
        if (mul) {
            ActF32::ld8(mul, (long long)n, C, c, t);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] *= t[j];
        }
        if (add) {
            ActF32::ld8(add, (long long)n, C, c, t);
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] += t[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            v[j] += r[j];
            v[j] = v[j] < 0.f ? 0.f : v[j];                               // nn.ReLU: NaN stays NaN
        }
        store8<A>(y, (long long)pix, C, c, v, ovf);
    }
}

// format: 0 bf16, 1 f16x3, 2 fp32
int plan(int N, int H, int W, int C, int format, orp_context_plan *out)
{
    if (!out || format < 0 || format > 2) return fail(ORP_EINVAL, "context_plan: needs a plan and format 0, 1 or 2");
    if (N < 1 || H < 1 || W < 1 || N > 65535 || (long long)H * W > 0x7fffffffLL)
        return fail(ORP_EINVAL, "context_pool: needs N, H, W >= 1, N <= 65535 and H * W < 2^31");
    if (C < 8 || C % 8 || C > kMaxC) return fail(ORP_EINVAL, "context_pool: C must be a multiple of 8 in [8, 2048]");
    const int wps = (C / 8 + 31) / 32;                 // warps per pixel slot
    const int slots = 8 / wps;
    const long long hw = (long long)H * W, pass = (long long)slots * kPix;
    long long chunks = (kTargetCtas + N - 1) / N;
    const long long most = (hw + pass - 1) / pass;      // at least one pass per chunk
    if (chunks > most) chunks = most;
    const long long L = (hw + chunks - 1) / chunks;
    chunks = (hw + L - 1) / L;                          // every chunk holds pixels
    *out = orp_context_plan{};
    out->threads = 32 * wps * slots;
    out->slots = slots;
    out->warps_per_slot = wps;
    out->chunks = (int)chunks;
    out->pixels_per_chunk = (int)L;
    out->grid_x = (int)chunks;
    out->grid_y = N;
    out->workspace_bytes = (long long)N * chunks * (C + 2) * (long long)sizeof(float);
    return ORP_OK;
}

template <class A>
int pool(const void *x, int N, int H, int W, int C, const float *mask_w, float *ws, size_t ws_bytes, void *stream, int format,
         const char *name)
{
    orp_context_plan pl;
    int rc = plan(N, H, W, C, format, &pl);
    if (rc) return rc;
    if (!x || !ws || !aligned16(x) || !aligned16(ws) || (mask_w && !aligned16(mask_w)))
        return fail(ORP_EINVAL, "%s: needs 16-byte aligned x, workspace and mask_w (NULL for 'avg')", name);
    if (ws_bytes < (size_t)pl.workspace_bytes) return fail(ORP_EINVAL, "%s: the workspace is smaller than the plan's workspace_bytes", name);
    if ((rc = ensure_device())) return rc;
    PoolP P{x, mask_w, ws, N, H * W, C, pl.chunks, pl.pixels_per_chunk, pl.slots, pl.warps_per_slot};
    context_pool_kernel<A><<<dim3(pl.grid_x, pl.grid_y), pl.threads, 0, static_cast<cudaStream_t>(stream)>>>(P);
    ORP_LAUNCHED();
    return ORP_OK;
}

bool mlp_ok(const orp_context_mlp *m)
{
    return m->w1 && m->b1 && m->ln_w && m->ln_b && m->w2 && m->b2 && aligned16(m->w1);
}

int transform(const float *ws, int N, int chunks, int C, int P, const orp_context_mlp *add_mlp, const orp_context_mlp *mul_mlp,
              float *add, float *mul, void *stream)
{
    if (!ws || N < 1 || chunks < 1 || chunks > kMaxChunks || C < 8 || C % 8 || C > kMaxC || P < 1 || P > kMaxC)
        return fail(ORP_EINVAL, "context_transform: needs the workspace, N >= 1, chunks in [1, 1024], C a multiple of 8 in [8, 2048] "
                                "and P in [1, 2048]");
    if (!add_mlp && !mul_mlp) return fail(ORP_EINVAL, "context_transform: needs at least one of add_mlp and mul_mlp");
    if ((add_mlp && (!add || !mlp_ok(add_mlp))) || (mul_mlp && (!mul || !mlp_ok(mul_mlp))))
        return fail(ORP_EINVAL, "context_transform: each given mlp needs all six tensors (w1 16-byte aligned) and its output");
    TransformP T{};
    T.ws = ws; T.N = N; T.chunks = chunks; T.C = C; T.P = P;
    int nf = 0;
    if (add_mlp) { T.mlp[nf] = *add_mlp; T.out[nf] = add; T.sigmoid[nf] = 0; ++nf; }
    if (mul_mlp) { T.mlp[nf] = *mul_mlp; T.out[nf] = mul; T.sigmoid[nf] = 1; ++nf; }
    int rc = ensure_device();
    if (rc) return rc;
    context_transform_kernel<<<dim3(N, nf), kTransformThreads, 0, static_cast<cudaStream_t>(stream)>>>(T);
    ORP_LAUNCHED();
    return ORP_OK;
}

template <class A>
int fuse(const void *x, const void *idt, int N, int H, int W, int C, const float *mul, const float *add, void *y, void *stream,
         const char *name)
{
    if (!x || !idt || !y || bad_dims(N, H, W, C) || !aligned16(x) || !aligned16(idt) || !aligned16(y) || y == x || y == idt)
        return fail(ORP_EINVAL, "%s: needs 16-byte aligned x, identity and a distinct y, N, H, W >= 1 and C a multiple of 8", name);
    if ((!mul && !add) || (mul && !aligned16(mul)) || (add && !aligned16(add)))
        return fail(ORP_EINVAL, "%s: needs 16-byte aligned mul and / or add (at least one)", name);
    unsigned int *ovf;
    int rc = overflow_ptr(A::planes == 2, ovf, name);
    if (rc || (rc = ensure_device())) return rc;
    context_fuse_kernel<A><<<grid_for((size_t)N * H * W * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const typename A::T *>(x), static_cast<const typename A::T *>(idt), N, H * W, C, mul, add,
        static_cast<typename A::T *>(y), ovf);
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace
}  // namespace orp

using namespace orp;

/* see include/orp_b200_context.h */
extern "C" int orp_context_make_plan(int N, int H, int W, int C, int format, orp_context_plan *out)
{
    return plan(N, H, W, C, format, out);
}

extern "C" int orp_context_pool_bf16(const void *x, int N, int H, int W, int C, const float *mask_w, float *workspace, size_t ws_bytes,
                                     void *stream)
{
    return pool<Act<false>>(x, N, H, W, C, mask_w, workspace, ws_bytes, stream, 0, "context_pool_bf16");
}
extern "C" int orp_context_pool_f16x3(const void *x, int N, int H, int W, int C, const float *mask_w, float *workspace, size_t ws_bytes,
                                      void *stream)
{
    return pool<Act<true>>(x, N, H, W, C, mask_w, workspace, ws_bytes, stream, 1, "context_pool_f16x3");
}
extern "C" int orp_context_pool_f32(const float *x, int N, int H, int W, int C, const float *mask_w, float *workspace, size_t ws_bytes,
                                    void *stream)
{
    return pool<ActF32>(x, N, H, W, C, mask_w, workspace, ws_bytes, stream, 2, "context_pool_f32");
}

extern "C" int orp_context_transform(const float *workspace, int N, int chunks, int C, int P, const orp_context_mlp *add_mlp,
                                     const orp_context_mlp *mul_mlp, float *add, float *mul, void *stream)
{
    return transform(workspace, N, chunks, C, P, add_mlp, mul_mlp, add, mul, stream);
}

extern "C" int orp_context_fuse_bf16(const void *x, const void *identity, int N, int H, int W, int C, const float *mul, const float *add,
                                     void *y, void *stream)
{
    return fuse<Act<false>>(x, identity, N, H, W, C, mul, add, y, stream, "context_fuse_bf16");
}
extern "C" int orp_context_fuse_f16x3(const void *x, const void *identity, int N, int H, int W, int C, const float *mul, const float *add,
                                      void *y, void *stream)
{
    return fuse<Act<true>>(x, identity, N, H, W, C, mul, add, y, stream, "context_fuse_f16x3");
}
extern "C" int orp_context_fuse_f32(const float *x, const float *identity, int N, int H, int W, int C, const float *mul, const float *add,
                                    float *y, void *stream)
{
    return fuse<ActF32>(x, identity, N, H, W, C, mul, add, y, stream, "context_fuse_f32");
}
