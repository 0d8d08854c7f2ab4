/*
 * orp_b200_group.h - C ABI of liborp_b200.so, continued: the grouped 3x3 convolution of ResNeXt backbones
 * (mmdet/models/backbones/resnext.py:44-54, conv2 = nn.Conv2d(width, width, 3, stride, 1, groups=groups, bias=False)).
 * Conventions (return codes, orp_last_error, device pointers, asynchronous on `stream`, orp_tc_problem, orp_tc_plan, the f16x3
 * operand format and its overflow count) are those of orp_b200.h.
 *
 * width = floor(planes * base_width / 64) * groups channels in and out, in groups of gw = width / groups channels: output
 * channel co reads input channels [gw * (co / gw), gw * (co / gw) + gw) only.  The tensor-core forms serve width % 64 == 0 and
 * gw in {4, 8, 16, 32, 64} (every published ResNeXt: 32x4d, 64x4d, 32x8d); anything else is ORP_EINVAL.  Every 64-channel
 * block of outputs reads the same 64-channel block of inputs; the tensor cores multiply only the max(16, gw)-wide diagonal
 * blocks of that 64 x 64 weight tile, max(16, gw) products per output channel and tap (gw of them useful).
 */
#ifndef ORP_B200_GROUP_H_
#define ORP_B200_GROUP_H_

#include "orp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* y = relu?(grouped_conv3x3(x, w, stride, pad 1) + bias) on the tensor cores, bf16 operands (the orp_conv2d_bf16 format).
 * Replaces nn.Conv2d(width, width, 3, stride, 1, groups=groups) + the folded bn2 + ReLU of resnext.py:44-54.
 *   prob   one problem: x bf16 NHWC [N,H,W,width], out bf16 NHWC [N,Ho,Wo,width]; residual_bf16, residual_f32, offset,
 *          gn_stats and mask must be NULL
 *   w      bf16 [width][9 taps][64]: the row of output channel co holds, per tap, the 64 input channels of its own 64-channel
 *          block (64 (co / 64) ..), the weights of its group in place and zero elsewhere
 *   bias   fp32 [width] or NULL; relu 0 / 1 */
int orp_group_conv2d_bf16(const orp_tc_problem *prob, const void *w, int width, int groups, int stride, const float *bias,
                          int relu, void *stream);
/* The same in f16x3 arithmetic (x and out split fp16 [N,H,W,2,width]); w fp16 [width][9 taps][2][64] holding (hi, lo) of
 * the weights of the bf16 layout times 2^wscale_log2 (0..15). */
int orp_group_conv2d_f16x3(const orp_tc_problem *prob, const void *w_split, int width, int groups, int stride,
                           const float *bias, int wscale_log2, int relu, void *stream);
/* The same on the CUDA cores in fp32: x fp32 NHWC [N,H,W,width], y fp32 NHWC [N,Ho,Wo,width], w fp32 [width][3][3][gw] (the
 * reference's [width, gw, 3, 3] with the input channels innermost).  Output channel co sums the 9 gw products of its group.
 * width % 4 == 0 and gw % 4 == 0 (float4 channel reads); any such groups, width. */
int orp_group_conv2d_f32(const float *x, int N, int H, int W, int width, int groups, const float *w, int stride,
                         const float *bias, int relu, float *y, void *stream);
/* Dry run: the plan (as orp_tc_last_plan would report it) of orp_group_conv2d_bf16 (split == 0) / _f16x3 (split != 0) over
 * probs on a device with `sms` SMs, with the same argument checks and error codes.  nprob != 1, out_f32 != 0, relu == 2 and
 * any residual / offset / mask / gn_stats pointer are ORP_EINVAL: the grouped walk serves conv2 alone.  Pointers are only
 * tested for NULL, never read; no device is needed, and the last-plan record is untouched. */
int orp_tc_plan_group_conv(int nprob, const orp_tc_problem *probs, const void *w, int width, int groups, int stride,
                           const float *bias, int relu, int out_f32, int split, int sms, orp_tc_plan *out);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_GROUP_H_ */
