// carafe.cu - the CARAFE top-down step of the FPN_CARAFE neck (include/orp_b200_carafe.h), in the three activation formats
// of the engines.
//
// One CTA per (tile of low-resolution pixels, image); the tile is kTileX pixels wide and `ty` rows high, clipped to the
// low-resolution pixels that have an output pixel inside the residual's extent.
//   1. The tile's logits (4 * G * k * k fp32 per pixel, contiguous) are copied to shared memory as float4 rows.
//   2. The softmax of each (output pixel, group) over its k * k taps runs in place, once, in fp32: the weights keep the
//      logits' layout, so the four sub-pixels' weights of a tap are one float4.
//   3. One item = (low-resolution pixel, 8 channels): the k x k window of x is read once for the item's four output pixels
//      (32 fp32 accumulators), then each output pixel inside the residual gets residual + sum and is stored.  A warp covers
//      the 256 channels of one pixel, so every tap is one contiguous row read; the tile's window overlaps hit L1.
// No float atomics: every sum has one order, so the results are bitwise reproducible.
#include <math.h>

#include "hrnet.cuh"
#include "../../include/orp_b200_carafe.h"

namespace orp {
namespace {

constexpr int kThreads = 256;
constexpr int kTileX = 8;                   // low-resolution pixels per tile row
constexpr int kMaxTileY = 4;
constexpr int kSmemBudget = 48 * 1024;      // the logits tile; no opt-in attribute needed

struct CarafeP {
    const void *x;
    const float *logits;
    const void *res;
    void *y;
    int N, H, W, C, Hr, Wr, G, Cl, ty, tiles_x;
    unsigned int *ovf;
};

template <class A, int K>
__global__ void __launch_bounds__(kThreads) carafe_add_kernel(const __grid_constant__ CarafeP P)
{
    extern __shared__ float4 s_logit4[];
    float *s_w = reinterpret_cast<float *>(s_logit4);
    constexpr int KK = K * K, R = (K - 1) / 2;
    const typename A::T *x = static_cast<const typename A::T *>(P.x);
    const typename A::T *res = static_cast<const typename A::T *>(P.res);
    typename A::T *y = static_cast<typename A::T *>(P.y);
    const int n = blockIdx.y;
    const int tx0 = (blockIdx.x % P.tiles_x) * kTileX, ty0 = (blockIdx.x / P.tiles_x) * P.ty;
    const int hl = (P.Hr + 1) >> 1, wl = (P.Wr + 1) >> 1;            // low-res pixels with an output inside the residual
    const int tw = min(kTileX, wl - tx0), th = min(P.ty, hl - ty0);
    const int lp = tw * th;
    const int cl4 = P.Cl >> 2;
    // 1. logits
    for (int i = threadIdx.x; i < lp * cl4; i += kThreads) {
        const int p = i / cl4, q = i - p * cl4;
        const int ly = ty0 + p / tw, lx = tx0 + p % tw;
        s_logit4[i] = reinterpret_cast<const float4 *>(P.logits + (((long long)n * P.H + ly) * P.W + lx) * P.Cl)[q];
    }
    __syncthreads();
    // 2. softmax over the k * k taps of (output pixel, group): item = (pixel, group, sub-pixel)
    for (int i = threadIdx.x; i < lp * 4 * P.G; i += kThreads) {
        const int sub = i & 3, pg = i >> 2;
        float *v = s_w + (pg / P.G) * P.Cl + (pg % P.G) * KK * 4 + sub;
        float m = -INFINITY;
#pragma unroll
        for (int t = 0; t < KK; ++t) m = fmaxf(m, v[4 * t]);
        float s = 0.f;
#pragma unroll
        for (int t = 0; t < KK; ++t) {
            const float e = expf(v[4 * t] - m);
            v[4 * t] = e;
            s += e;
        }
#pragma unroll
        for (int t = 0; t < KK; ++t) v[4 * t] = v[4 * t] / s;
    }
    __syncthreads();
    // 3. reassembly + residual
    const int c8 = P.C >> 3, cpg = P.C / P.G;
    for (int i = threadIdx.x; i < lp * c8; i += kThreads) {
        const int p = i / c8, c = (i - p * c8) * 8;
        const int ly = ty0 + p / tw, lx = tx0 + p % tw;
        const float4 *w4 = s_logit4 + (p * P.Cl + (c / cpg) * KK * 4) / 4;
        float acc[4][8];
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[s][j] = 0.f;
#pragma unroll
        for (int dy = 0; dy < K; ++dy) {
            const int iy = ly + dy - R;
            if (iy < 0 || iy >= P.H) continue;
#pragma unroll
            for (int dx = 0; dx < K; ++dx) {
                const int ix = lx + dx - R;
                if (ix < 0 || ix >= P.W) continue;
                float v[8];
                A::ld8(x, ((long long)n * P.H + iy) * P.W + ix, P.C, c, v);
                const float4 w = w4[dy * K + dx];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    acc[0][j] = fmaf(w.x, v[j], acc[0][j]);
                    acc[1][j] = fmaf(w.y, v[j], acc[1][j]);
                    acc[2][j] = fmaf(w.z, v[j], acc[2][j]);
                    acc[3][j] = fmaf(w.w, v[j], acc[3][j]);
                }
            }
        }
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int oy = 2 * ly + (s >> 1), ox = 2 * lx + (s & 1);
            if (oy >= P.Hr || ox >= P.Wr) continue;
            const long long tok = ((long long)n * P.Hr + oy) * P.Wr + ox;
            float r[8];
            A::ld8(res, tok, P.C, c, r);
#pragma unroll
            for (int j = 0; j < 8; ++j) r[j] += acc[s][j];
            store8<A>(y, tok, P.C, c, r, P.ovf);
        }
    }
}

template <class A>
int carafe_add(const void *x, int N, int H, int W, int C, const float *logits, int k, int G, const void *res, int Hr, int Wr,
               void *y, void *stream, const char *name)
{
    if (!x || !logits || !res || !y || !aligned16(x) || !aligned16(logits) || !aligned16(res) || !aligned16(y) || y == x ||
        y == res)
        return fail(ORP_EINVAL, "%s: needs 16-byte aligned x, logits, residual and a y distinct from x and the residual", name);
    if (bad_dims(N, H, W, C) || N > 65535)
        return fail(ORP_EINVAL, "%s: needs N in [1, 65535], H, W >= 1 and C a multiple of 8", name);
    if ((k != 1 && k != 3 && k != 5 && k != 7) || (G != 1 && G != 2 && G != 4) || (C / G) % 8 || C % G)
        return fail(ORP_EINVAL, "%s: needs up_kernel k in {1, 3, 5, 7}, up_group G in {1, 2, 4} and C / G a multiple of 8", name);
    if (Hr < 1 || Wr < 1 || Hr > 2 * H || Wr > 2 * W)
        return fail(ORP_EINVAL, "%s: the residual's Hr, Wr must lie in [1, 2H] and [1, 2W]", name);
    const int cl = 4 * G * k * k;
    int ty = kSmemBudget / (kTileX * cl * (int)sizeof(float));
    ty = ty < 1 ? 1 : (ty > kMaxTileY ? kMaxTileY : ty);
    const int hl = (Hr + 1) / 2, wl = (Wr + 1) / 2;
    const int tiles_x = (wl + kTileX - 1) / kTileX, tiles_y = (hl + ty - 1) / ty;
    if ((long long)tiles_x * tiles_y > 0x7fffffffLL) return fail(ORP_EINVAL, "%s: the map is too large", name);
    CarafeP P{x, logits, res, y, N, H, W, C, Hr, Wr, G, cl, ty, tiles_x, nullptr};
    int rc = overflow_ptr(A::planes == 2, P.ovf, name);
    if (rc || (rc = ensure_device())) return rc;
    const dim3 grid(tiles_x * tiles_y, N);
    const size_t smem = (size_t)kTileX * ty * cl * sizeof(float);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (k) {
    case 1: carafe_add_kernel<A, 1><<<grid, kThreads, smem, st>>>(P); break;
    case 3: carafe_add_kernel<A, 3><<<grid, kThreads, smem, st>>>(P); break;
    case 5: carafe_add_kernel<A, 5><<<grid, kThreads, smem, st>>>(P); break;
    default: carafe_add_kernel<A, 7><<<grid, kThreads, smem, st>>>(P); break;
    }
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace
}  // namespace orp

using namespace orp;

/* see include/orp_b200_carafe.h */
extern "C" int orp_carafe_add_bf16(const void *x, int N, int H, int W, int C, const float *logits, int k, int G, const void *residual,
                                   int Hr, int Wr, void *y, void *stream)
{
    return carafe_add<Act<false>>(x, N, H, W, C, logits, k, G, residual, Hr, Wr, y, stream, "carafe_add_bf16");
}
extern "C" int orp_carafe_add_f16x3(const void *x, int N, int H, int W, int C, const float *logits, int k, int G, const void *residual,
                                    int Hr, int Wr, void *y, void *stream)
{
    return carafe_add<Act<true>>(x, N, H, W, C, logits, k, G, residual, Hr, Wr, y, stream, "carafe_add_f16x3");
}
extern "C" int orp_carafe_add_f32(const float *x, int N, int H, int W, int C, const float *logits, int k, int G, const float *residual,
                                  int Hr, int Wr, float *y, void *stream)
{
    return carafe_add<ActF32>(x, N, H, W, C, logits, k, G, residual, Hr, Wr, y, stream, "carafe_add_f32");
}
