/*
 * orp_b200_attention.h - C ABI of liborp_b200.so, continued: the generalized ("empirical") attention block of ResNet
 * backbones (mmdet/ops/generalized_attention.py, "An Empirical Study of Spatial Attention Mechanisms in Deep Networks"),
 * spatial_range = -1, q_stride = 1.  Conventions (return codes, orp_last_error, device pointers, asynchronous on `stream`,
 * the bf16 and f16x3 activation formats) are those of orp_b200.h.  Every tensor is NHWC with C innermost (f16x3: fp16
 * [.., 2, C], the C hi values then the C lo values).  Softmax and accumulation are fp32 in every format.
 *
 * The block on x [N, C, H, W], head dimension d = C / heads, kv_stride s (1 or 2), Hk = ceil(H / s), Wk = ceil(W / s):
 *   energy(q, k) = Qc[q] . K[k] + Qp[q] . (Px[qx - s kx] + Py[qy - s ky])        per head, no 1/sqrt(d) scale
 *   out[q]       = sum_k softmax_k(energy(q, k)) V[k]
 * with Qc = [t0] query + [t2] appr_bias and Qp = [t1] query + [t3] geom_bias for attention_type t, K and V the 1x1
 * convolutions of x[:, :, ::s, ::s], and Px / Py the position tables appr_geom_fc_{x,y}(embedding(offset)) / sqrt(2).
 * The entry points below compute `out` from Qc, Qp, K, V and the tables; the 1x1 convolutions around them are the library's
 * convolutions.
 */
#ifndef ORP_B200_ATTENTION_H_
#define ORP_B200_ATTENTION_H_

#include "orp_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* One attention launch.  Token t of a [.., C']-channel tensor holds channel c at element t * ld + c (f16x3: the hi value
 * there, the lo value ld elements further, token pitch 2 ld); the pointers below point at the first channel of head 0 of
 * token 0, so several operands may live in one tensor at different channel offsets (multiples of 8).
 *   q_c     Qc of the H * W queries of each image, pitch ld_q; NULL: no content term (k must then be NULL too)
 *   q_p     Qp, pitch ld_q; NULL: no position term (pos_x, pos_y must then be NULL too)
 *   k, v    K and V of the Hk * Wk keys of each image in raster order, pitch ld_kv
 *   pos_x   Px, Rx = W + s (Wk - 1) rows of C channels (pitch C): row r is the x offset r - s (Wk - 1)
 *   pos_y   Py, Ry = H + s (Hk - 1) rows of C channels: row r is the y offset r - s (Hk - 1)
 *   out     [N, H, W, C], distinct from every input
 * With a position term Hk and Wk must be ceil(H / s) and ceil(W / s); without one they are free (the '0010' shortcut runs
 * one query per image, H = W = 1, against the full key map). */
typedef struct orp_gen_attention_args {
    const void *q_c, *q_p, *k, *v, *pos_x, *pos_y;
    void *out;
    int N, H, W, Hk, Wk, kv_stride, C, heads, ld_q, ld_kv;
} orp_gen_attention_args;

/* What a launch runs: one CTA of `threads` threads per (query tile of queries_per_cta, head, image) = grid (x, y, z), with
 * smem_bytes of dynamic shared memory; rx / ry position-table rows (0 without a position term). */
typedef struct orp_gen_attention_plan {
    int head_dim, queries_per_cta, threads, grid_x, grid_y, grid_z, smem_bytes, rx, ry, content, position;
} orp_gen_attention_plan;

/* Tensor cores (mma.sync m16n8k16, fp32 accumulation), bf16 operands. */
int orp_gen_attention_bf16(const orp_gen_attention_args *a, void *stream);
/* Tensor cores in f16x3 arithmetic: every product hi*hi + lo*hi + hi*lo of fp16 pairs, tables in the split format. */
int orp_gen_attention_f16x3(const orp_gen_attention_args *a, void *stream);
/* CUDA cores, fp32 tensors throughout. */
int orp_gen_attention_f32(const orp_gen_attention_args *a, void *stream);

/* Dry run: the plan of orp_gen_attention_bf16 (format 0), _f16x3 (1) or _f32 (2), with the same argument checks and error
 * codes.  Accepted: N, H, W, Hk, Wk >= 1, N <= 65535, heads <= 65535, C = heads * d with d 32 or 64, kv_stride 1 or 2,
 * ld_q and ld_kv multiples of 8 and >= C, 16-byte aligned pointers, out and v not NULL, the NULL pairings above, and the
 * shared memory of the launch within the 227 KiB of an sm_90 CTA (the per-query position rows grow with Hk + Wk).
 * Pointers are tested, never read; no device is needed. */
int orp_gen_attention_make_plan(const orp_gen_attention_args *a, int format, orp_gen_attention_plan *out);

/* The '0010' shortcut's last step: y[n, h, w, c] = x[n, h, w, c] + row[n, c].  x, y [N, H, W, C] in the entry point's
 * format (distinct), row fp32 [N, C] (gamma * proj_conv of the attended row); C % 8 == 0. */
int orp_gen_attention_bcast_add_bf16(const void *x, int N, int H, int W, int C, const float *row, void *y, void *stream);
int orp_gen_attention_bcast_add_f16x3(const void *x, int N, int H, int W, int C, const float *row, void *y, void *stream);
int orp_gen_attention_bcast_add_f32(const float *x, int N, int H, int W, int C, const float *row, float *y, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_ATTENTION_H_ */
