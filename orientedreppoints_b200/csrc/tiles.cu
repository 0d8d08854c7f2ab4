// tiles.cu - tile producer on the device (SURVEY §8 row n4).
// Test infrastructure it is not: this is the product path that replaces
// DOTA_devkit/SplitOnlyImage_multi_process.py:38-49 (saveimagepatches: crop subsize x subsize at (left, up), zero
// padded to the full tile) - the reference writes every tile to a PNG and the data loader decodes it again; here the
// decoded image is uploaded once and the batch of uint8 HWC tiles the detector consumes is cut out in HBM.
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"

namespace orp {
namespace {

// one thread = 4 output bytes (out rows are subsize*C bytes, a multiple of 4 is required by the host wrapper)
__global__ void __launch_bounds__(256)
split_tiles_kernel(const uint8_t *__restrict__ img, int H, int W, int C, const int32_t *__restrict__ origins, int ntiles,
                   int subsize, uint8_t *__restrict__ out)
{
    const size_t row_bytes = (size_t)subsize * C;
    const size_t words_per_row = row_bytes / 4, words_per_tile = words_per_row * subsize;
    const size_t total = words_per_tile * ntiles;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int t = (int)(i / words_per_tile);
        const size_t r = i - (size_t)t * words_per_tile;
        const int y = (int)(r / words_per_row);
        const int xb = (int)(r - (size_t)y * words_per_row) * 4;           // byte offset inside the tile row
        const int left = origins[2 * t], up = origins[2 * t + 1];
        const int sy = up + y;
        const int valid_bytes = (W - left < subsize ? W - left : subsize) * C;   // bytes of this row that come from the image
        uint32_t v = 0;
        if (sy < H && xb < valid_bytes) {
            const uint8_t *src = img + ((size_t)sy * W + left) * C + xb;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (xb + k < valid_bytes) v |= (uint32_t)src[k] << (8 * k);
        }
        reinterpret_cast<uint32_t *>(out)[i] = v;
    }
}

}  // namespace
}  // namespace orp

extern "C" int orp_split_tiles_u8(const uint8_t *img_hwc, int H, int W, int C, const int32_t *origins, int ntiles, int subsize,
                                  uint8_t *out, void *stream)
{
    using namespace orp;
    if (!img_hwc || !origins || !out || H < 1 || W < 1 || C < 1 || ntiles < 0 || subsize < 1 || ((size_t)subsize * C) % 4)
        return fail(ORP_EINVAL, "orp_split_tiles_u8: bad arguments (subsize*C must be a multiple of 4)");
    int rc = ensure_device();
    if (rc) return rc;
    if (ntiles == 0) return ORP_OK;
    const size_t total = (size_t)ntiles * subsize * ((size_t)subsize * C / 4);
    split_tiles_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(img_hwc, H, W, C, origins, ntiles,
                                                                                           subsize, out);
    ORP_LAUNCHED();
    return ORP_OK;
}
