/*
 * orp_b200_carafe.h - C ABI of liborp_b200.so, continued: the top-down step of the FPN_CARAFE neck, content-aware
 * reassembly of features (CARAFE, "CARAFE: Content-Aware ReAssembly of FEatures", ICCV 2019; mmdet/ops/carafe CARAFEPack,
 * mmdet/models/necks/fpn_carafe.py) with scale factor 2, fused with the top-down add.
 * Conventions (return codes, orp_last_error, device pointers, asynchronous on `stream`, the bf16 and f16x3 activation
 * formats) are those of orp_b200.h.  Every activation is NHWC with C innermost (f16x3: fp16 [.., 2, C], the C hi values then
 * the C lo values).
 *
 * On x [N, H, W, C], the content encoder's fp32 logits [N, H, W, 4 * G * k * k] and a residual [N, Hr, Wr, C] with
 * 1 <= Hr <= 2H, 1 <= Wr <= 2W, one launch writes y [N, Hr, Wr, C]:
 *   w[n, oy, ox, g, t] = softmax_t(logits[n, oy / 2, ox / 2, (g * k * k + t) * 4 + (oy % 2) * 2 + (ox % 2)]), t < k * k
 *   y[n, oy, ox, c]    = residual[n, oy, ox, c]
 *                        + sum_{t = (i, j) inside the map} w[n, oy, ox, c / (C / G), t] x[n, oy / 2 + i - r, ox / 2 + j - r, c]
 * with r = (k - 1) / 2: pixel_shuffle(2) of the logits, the softmax over all k * k taps, the reassembly in which taps outside
 * x are skipped (not renormalised, so border outputs carry a total weight below 1), and the add of the finer lateral, cut to
 * its extent (fpn_carafe.py slice_as).  Each output pixel's softmax is computed once, in fp32, for all its channels; the
 * four output pixels of a low-resolution pixel share one read of its k x k window.  No atomics on the data: results are
 * bitwise reproducible.
 */
#ifndef ORP_B200_CARAFE_H_
#define ORP_B200_CARAFE_H_

#include "orp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* x, residual and y in the entry point's format (y distinct from both), logits fp32, every pointer 16-byte aligned.
 * Accepted: N, H, W >= 1, N <= 65535, C a multiple of 8 with C / G a multiple of 8, k (up_kernel) in {1, 3, 5, 7},
 * G (up_group) in {1, 2, 4}, 1 <= Hr <= 2H, 1 <= Wr <= 2W; anything else returns ORP_EINVAL before any launch.
 * The f16x3 stores saturate and are counted by orp_f16x3_overflow_count. */
int orp_carafe_add_bf16(const void *x, int N, int H, int W, int C, const float *logits, int k, int G, const void *residual,
                        int Hr, int Wr, void *y, void *stream);
int orp_carafe_add_f16x3(const void *x, int N, int H, int W, int C, const float *logits, int k, int G, const void *residual,
                         int Hr, int Wr, void *y, void *stream);
int orp_carafe_add_f32(const float *x, int N, int H, int W, int C, const float *logits, int k, int G, const float *residual,
                       int Hr, int Wr, float *y, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_CARAFE_H_ */
