// hrnet.cu - the tensor-core engines' HRNet / HRFPN layers (include/orp_b200_hrnet.h): the kernels of hrnet.cuh in the bf16
// and f16x3 activation formats.  The fp32 forms are in dense_f32.cu.
#include "hrnet.cuh"
#include "../../include/orp_b200_hrnet.h"

using namespace orp;

/* see include/orp_b200_hrnet.h */
extern "C" int orp_hr_fuse_bf16(const void *base, int N, int H, int W, int C, int nsrc, const void *const *src, void *y, void *stream)
{
    return hr_fuse<Act<false>>(base, N, H, W, C, nsrc, src, y, stream, "hr_fuse_bf16");
}

extern "C" int orp_hr_fuse_f16x3(const void *base, int N, int H, int W, int C, int nsrc, const void *const *src, void *y, void *stream)
{
    return hr_fuse<Act<true>>(base, N, H, W, C, nsrc, src, y, stream, "hr_fuse_f16x3");
}

extern "C" int orp_hrfpn_reduce_bf16(int nparts, const float *const *part, int N, int H, int W, int C, void *y, void *stream)
{
    return hrfpn_reduce<Act<false>>(nparts, part, N, H, W, C, y, stream, "hrfpn_reduce_bf16");
}

extern "C" int orp_hrfpn_reduce_f16x3(int nparts, const float *const *part, int N, int H, int W, int C, void *y, void *stream)
{
    return hrfpn_reduce<Act<true>>(nparts, part, N, H, W, C, y, stream, "hrfpn_reduce_f16x3");
}

extern "C" int orp_hrfpn_pool_bf16(const void *x, int N, int H, int W, int C, int max_pool, void *const *out, void *stream)
{
    return hrfpn_pool<Act<false>>(x, N, H, W, C, max_pool, out, stream, "hrfpn_pool_bf16");
}

extern "C" int orp_hrfpn_pool_f16x3(const void *x, int N, int H, int W, int C, int max_pool, void *const *out, void *stream)
{
    return hrfpn_pool<Act<true>>(x, N, H, W, C, max_pool, out, stream, "hrfpn_pool_f16x3");
}
