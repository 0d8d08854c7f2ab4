/*
 * orp_b200_swin.h - C ABI of liborp_b200.so, continued: the kernels the Swin-S / Swin-B / Swin-L backbones need beyond
 * Swin-T's (mmdet/models/backbones/swin_transformer.py:449-631 with window_size 12 or embed_dim 128 / 192).  Conventions
 * (return codes, orp_last_error, device pointers, asynchronous on `stream`, the bf16 and f16x3 token formats) are those of
 * orp_b200.h; the parameters are those of orp_window_attention_* and orp_layernorm_*.
 */
#ifndef ORP_B200_SWIN_H_
#define ORP_B200_SWIN_H_

#ifdef __cplusplus
extern "C" {
#endif

/* (shifted) 12x12 window attention with relative position bias and the -100 region mask (WindowAttention.forward :122-154,
 * BasicLayer mask :371-390): qkv [B,Hp,Wp,3C] (q|k|v, heads x 32), bias_table fp32 [529, heads]; out [B,H,W,C] at the original
 * token positions.  Requires Hp % 12 == 0, Wp % 12 == 0, 0 <= shift < 12 and heads * 32 == C. */
int orp_window_attention12_bf16(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                const float *bias_table, float scale, void *out, void *stream);
int orp_window_attention12_f16x3(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                 const float *bias_table, float scale, void *out, void *stream);
/* LayerNorm over 1536 < C <= 3072 channels, C % 8 == 0 (the PatchMerging norms of Swin-B stage 2 and Swin-L stages 1-2);
 * x [B,H,W,C] -> y [B,Hp,Wp,C] (H x W interior written), as orp_layernorm_*, which covers C <= 1536. */
int orp_layernorm_wide_bf16(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps,
                            int Hp, int Wp, void *y, void *stream);
int orp_layernorm_wide_f16x3(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps,
                             int Hp, int Wp, void *y, void *stream);

#ifdef __cplusplus
}
#endif

#endif /* ORP_B200_SWIN_H_ */
