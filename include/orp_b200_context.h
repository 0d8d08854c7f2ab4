/*
 * orp_b200_context.h - C ABI of liborp_b200.so, continued: the global context block (GCB) of GCNet in ResNet / ResNeXt
 * bottlenecks (mmdet/ops/context_block.py, "GCNet: Non-local Networks Meet Squeeze-Excitation Networks and Beyond").
 * Conventions (return codes, orp_last_error, device pointers, asynchronous on `stream`, the bf16 and f16x3 activation
 * formats) are those of orp_b200.h.  Every activation is NHWC with C innermost (f16x3: fp16 [.., 2, C], the C hi values then
 * the C lo values).  Every reduction is fp32 in a fixed order, without atomics: results are bitwise reproducible.
 *
 * The block on x [N, C, H, W] (the bottleneck's bn3(conv3(.)), before the residual add), P = int(C * ratio):
 *   'att':  ctx[n]  = sum_p softmax_p(w_mask . x[n, p]) x[n, p]        (conv_mask's bias cancels in the softmax)
 *   'avg':  ctx[n]  = mean_p x[n, p]
 *   t       = W2 relu(LayerNorm_P(W1 ctx + b1)) + b2                    per fusion (channel_add_conv / channel_mul_conv)
 *   y[n, p] = relu(x[n, p] * sigmoid(t_mul[n]) + t_add[n] + identity[n, p])
 * as three launches: a pool into per-chunk partials (x read once), one transform per block (the chunks combined in a fixed
 * order, then the MLPs), and one fuse pass.  Partials of chunk j of image n: the chunk's logit maximum m, its sum of
 * exp(logit - m) (the pixel count for 'avg') and its exp-weighted sum of x, all fp32.
 */
#ifndef ORP_B200_CONTEXT_H_
#define ORP_B200_CONTEXT_H_

#include <stddef.h>

#include "orp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* What a pool launch runs: one CTA of `threads` threads per (chunk of pixels_per_chunk pixels, image) = grid (chunks, N).
 * The CTA holds `slots` pixel slots of warps_per_slot warps (8 channels per lane) and reads 4 pixels per slot at a time.
 * workspace_bytes: the fp32 partials the caller provides, N * chunks * (C + 2) floats. */
typedef struct orp_context_plan {
    int threads, slots, warps_per_slot, chunks, pixels_per_chunk, grid_x, grid_y;
    long long workspace_bytes;
} orp_context_plan;

/* Dry run: the plan of the pool launch of orp_context_pool_bf16 (format 0), _f16x3 (1) or _f32 (2) on x [N, H, W, C], with
 * the same argument checks and error codes.  Accepted: N, H, W >= 1, N <= 65535, H * W < 2^31, C a multiple of 8 in
 * [8, 2048].  The grid aims at 528 CTAs (four per SM of an H100 SXM): ceil(528 / N) chunks per image, fewer when the map
 * holds fewer passes of a CTA (slots * 4 pixels each), so it covers the 132 SMs whenever N * H * W holds 132 such passes -
 * every stage of a ResNet at N = 1 on 960^2 and 1024^2 input.  No device is needed. */
int orp_context_make_plan(int N, int H, int W, int C, int format, orp_context_plan *out);

/* Pool: x [N, H, W, C] in the entry point's format; mask_w fp32 [C], the conv_mask weight ('att'), or NULL for 'avg';
 * workspace fp32, at least the plan's workspace_bytes (ws_bytes), 16-byte aligned like x. */
int orp_context_pool_bf16(const void *x, int N, int H, int W, int C, const float *mask_w, float *workspace, size_t ws_bytes,
                          void *stream);
int orp_context_pool_f16x3(const void *x, int N, int H, int W, int C, const float *mask_w, float *workspace, size_t ws_bytes,
                           void *stream);
int orp_context_pool_f32(const float *x, int N, int H, int W, int C, const float *mask_w, float *workspace, size_t ws_bytes,
                         void *stream);

/* One fusion's MLP, fp32, in the reference's layouts: w1 [P, C], b1 [P], ln_w / ln_b [P] (LayerNorm([P, 1, 1]), eps 1e-5),
 * w2 [C, P], b2 [C]. */
typedef struct orp_context_mlp {
    const float *w1, *b1, *ln_w, *ln_b, *w2, *b2;
} orp_context_mlp;

/* Transform, one launch for every format, on the CUDA cores: the `chunks` partials per image of a pool launch -> the
 * context -> add[n, c] = t_add (add_mlp) and mul[n, c] = sigmoid(t_mul) (mul_mlp), fp32 [N, C].  A NULL mlp leaves its
 * output unwritten (and it may be NULL); at least one is given.  C % 8 == 0, C and P in [1, 2048], chunks in [1, 1024]. */
int orp_context_transform(const float *workspace, int N, int chunks, int C, int P, const orp_context_mlp *add_mlp,
                          const orp_context_mlp *mul_mlp, float *add, float *mul, void *stream);

/* Fuse: y = relu(x * mul[n, c] + add[n, c] + identity), x / identity / y [N, H, W, C] in the entry point's format (y distinct
 * from both), mul / add fp32 [N, C] (NULL: no such term; at least one is given).  C % 8 == 0.  The f16x3 stores saturate and
 * are counted by orp_f16x3_overflow_count. */
int orp_context_fuse_bf16(const void *x, const void *identity, int N, int H, int W, int C, const float *mul, const float *add,
                          void *y, void *stream);
int orp_context_fuse_f16x3(const void *x, const void *identity, int N, int H, int W, int C, const float *mul, const float *add,
                           void *y, void *stream);
int orp_context_fuse_f32(const float *x, const float *identity, int N, int H, int W, int C, const float *mul, const float *add,
                         float *y, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_CONTEXT_H_ */
