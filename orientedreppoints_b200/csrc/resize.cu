// resize.cu - the test pipeline's Resize (+ RandomFlip, + Pad) on the device.
// mmcv.imrescale -> imresize -> cv2.resize(INTER_LINEAR) on uint8 HWC images (configs/dota/*.py test_pipeline:
// RotateResize(keep_ratio=True) -> RotateRandomFlip -> Normalize -> Pad(size_divisor=32)).  cv2's uint8 bilinear path is
// integer arithmetic once its per-column / per-row coefficients exist; those are computed on the host in float32 exactly
// as cv2 does (orientedreppoints_b200/datasets/pipelines.py: resize_tables) and passed in as two small tables, so this
// kernel is integer-only and bit-identical to cv2:
//   horizontal:  h = S[r][sx0] * a0 + S[r][sx1] * a1                         (int, coefficients scaled by 2048)
//   vertical:    d = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2, saturated to uint8
// xtab: int32 [Wd][4] = (sx0, sx1, a0, a1), columns already clamped into [0, W-1];
// ytab: int32 [Hd][4] = (r0, r1, b0, b1), rows already clamped into [0, H-1].
// Mirroring (flip) is applied after the resize, as RandomFlip follows Resize; the two orders differ bit for bit.  Output
// pixels outside [Hd, Wd] of the [Hp, Wp] destination are written as 0 (Normalize follows, so the stems mask them out).
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace orp {
namespace {

template <int C>
__global__ void __launch_bounds__(256)
resize_u8_kernel(const uint8_t *__restrict__ src, int H, int W, uint8_t *__restrict__ dst, int Hd, int Wd, int Hp, int Wp,
                 int flip, const int4 *__restrict__ xtab, const int4 *__restrict__ ytab)
{
    const int row = blockIdx.y;                     // n * Hp + y
    const int n = row / Hp, y = row - n * Hp;
    uint8_t *drow = dst + (size_t)row * Wp * C;
    if (y >= Hd) {
        for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < Wp; x += gridDim.x * blockDim.x)
#pragma unroll
            for (int c = 0; c < C; ++c) drow[x * C + c] = 0;
        return;
    }
    const int4 yt = ytab[y];
    const uint8_t *s0 = src + ((size_t)n * H + yt.x) * W * C, *s1 = src + ((size_t)n * H + yt.y) * W * C;
    for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < Wp; x += gridDim.x * blockDim.x) {
        if (x >= Wd) {
#pragma unroll
            for (int c = 0; c < C; ++c) drow[x * C + c] = 0;
            continue;
        }
        const int4 xt = xtab[flip ? Wd - 1 - x : x];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int h0 = (int)s0[xt.x * C + c] * xt.z + (int)s0[xt.y * C + c] * xt.w;
            const int h1 = (int)s1[xt.x * C + c] * xt.z + (int)s1[xt.y * C + c] * xt.w;
            int v = (((yt.z * (h0 >> 4)) >> 16) + ((yt.w * (h1 >> 4)) >> 16) + 2) >> 2;
            drow[x * C + c] = (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        }
    }
}

template <int C>
void launch(const uint8_t *src, int N, int H, int W, uint8_t *dst, int Hd, int Wd, int Hp, int Wp, int flip, const int32_t *xtab,
            const int32_t *ytab, cudaStream_t stream)
{
    const dim3 grid((unsigned)((Wp + 255) / 256), (unsigned)(N * Hp));
    resize_u8_kernel<C><<<grid, 256, 0, stream>>>(src, H, W, dst, Hd, Wd, Hp, Wp, flip, reinterpret_cast<const int4 *>(xtab),
                                                  reinterpret_cast<const int4 *>(ytab));
}

}  // namespace
}  // namespace orp

extern "C" int orp_resize_u8(const uint8_t *src, int N, int H, int W, int C, uint8_t *dst, int Hd, int Wd, int Hp, int Wp, int flip,
                             const int32_t *xtab, const int32_t *ytab, void *stream)
{
    using namespace orp;
    if (!src || !dst || !xtab || !ytab || N < 0 || H < 1 || W < 1 || C < 1 || C > 4 || Hd < 1 || Wd < 1 || Hp < Hd || Wp < Wd ||
        Hp > 65535 || ((uintptr_t)xtab & 15) || ((uintptr_t)ytab & 15))
        return fail(ORP_EINVAL, "orp_resize_u8: bad arguments (1 <= C <= 4, Hd <= Hp <= 65535, Wd <= Wp, 16-byte aligned tables)");
    int rc = ensure_device();
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int per = 65535 / Hp;                     // gridDim.y holds at most 65535 rows: launch in slices of whole images
    for (int n0 = 0; n0 < N; n0 += per) {
        const int nn = N - n0 < per ? N - n0 : per;
        const uint8_t *s = src + (size_t)n0 * H * W * C;
        uint8_t *d = dst + (size_t)n0 * Hp * Wp * C;
        switch (C) {
        case 1: launch<1>(s, nn, H, W, d, Hd, Wd, Hp, Wp, flip, xtab, ytab, st); break;
        case 2: launch<2>(s, nn, H, W, d, Hd, Wd, Hp, Wp, flip, xtab, ytab, st); break;
        case 3: launch<3>(s, nn, H, W, d, Hd, Wd, Hp, Wp, flip, xtab, ytab, st); break;
        default: launch<4>(s, nn, H, W, d, Hd, Wd, Hp, Wp, flip, xtab, ytab, st); break;
        }
        ORP_LAUNCHED();
    }
    return ORP_OK;
}
