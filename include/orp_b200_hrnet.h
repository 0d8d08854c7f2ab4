/*
 * orp_b200_hrnet.h - C ABI of liborp_b200.so, continued: the memory-bound layers of HRNet backbones and their HRFPN neck
 * (mmdet/models/backbones/hrnet.py, mmdet/models/necks/hrfpn.py).  Conventions (return codes, orp_last_error, device
 * pointers, asynchronous on `stream`, the bf16 and f16x3 activation formats and the f16x3 overflow count) are those of
 * orp_b200.h.  Every tensor is NHWC with C innermost (f16x3: fp16 [.., 2, C], the C hi values then the C lo values); every
 * f16x3 output beyond the fp16 range saturates and is counted in orp_f16x3_overflow_count.  All arithmetic is fp32.
 *
 * Accepted arguments, for every entry point: N, H, W >= 1, C >= 8 and C % 8 == 0 (16-byte channel vectors), no NULL
 * pointer among those used, and the extents named below; anything else returns ORP_EINVAL before any launch.
 */
#ifndef ORP_B200_HRNET_H_
#define ORP_B200_HRNET_H_

#include "orp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The fusion of one HRModule output branch (hrnet.py:182-190) after the down-sampling terms: y = relu(base + sum over
 * k = 1..nsrc of nearest_up(src[k - 1], 2^k)).
 *   base   [N,H,W,C]: x_i plus every stride-2 down-chain term of the lower branches j < i
 *   src    host array of nsrc (1..3) device pointers; src[k - 1] is [N, H / 2^k, W / 2^k, C], the 1x1 conv + BN of branch
 *          i + k at its own resolution (H and W multiples of 2^nsrc)
 *   y      [N,H,W,C], distinct from every input */
int orp_hr_fuse_bf16(const void *base, int N, int H, int W, int C, int nsrc, const void *const *src, void *y, void *stream);
int orp_hr_fuse_f16x3(const void *base, int N, int H, int W, int C, int nsrc, const void *const *src, void *y, void *stream);
int orp_hr_fuse_f32(const float *base, int N, int H, int W, int C, int nsrc, const float *const *src, float *y, void *stream);

/* HRFPN's bilinear upsampling, concatenation and 1x1 reduction (hrfpn.py:80-88), with the 1x1 applied first:
 * y = sum over i = 0..nparts-1 of bilinear_up(part[i], 2^i), F.interpolate(scale_factor=2^i, mode='bilinear',
 * align_corners=False), summed in the order i = 0, 1, ...
 *   part   host array of nparts (1..4) device pointers, fp32 [N, H / 2^i, W / 2^i, C]: branch i times its column slice of
 *          reduction_conv (the bias is in part[0]); H and W multiples of 2^(nparts-1)
 *   y      [N,H,W,C] in the entry point's activation format (fp32 for _f32) */
int orp_hrfpn_reduce_bf16(int nparts, const float *const *part, int N, int H, int W, int C, void *y, void *stream);
int orp_hrfpn_reduce_f16x3(int nparts, const float *const *part, int N, int H, int W, int C, void *y, void *stream);
int orp_hrfpn_reduce_f32(int nparts, const float *const *part, int N, int H, int W, int C, float *y, void *stream);

/* HRFPN's pooled pyramid (hrfpn.py:89-91) in one pass over x: out[l - 1] = avg_pool2d / max_pool2d(x, 2^l, 2^l) for
 * l = 1..4, [N, H / 2^l, W / 2^l, C] rounded down: a partial window is dropped, as torch drops it.
 *   max_pool   0: average (the sum of the 4^l values times 4^-l), 1: maximum
 *   out        host array of 4 device pointers; a level whose extent rounds to 0 is not written (its pointer may be NULL) */
int orp_hrfpn_pool_bf16(const void *x, int N, int H, int W, int C, int max_pool, void *const *out, void *stream);
int orp_hrfpn_pool_f16x3(const void *x, int N, int H, int W, int C, int max_pool, void *const *out, void *stream);
int orp_hrfpn_pool_f32(const float *x, int N, int H, int W, int C, int max_pool, float *const *out, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_HRNET_H_ */
