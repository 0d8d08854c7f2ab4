// swin.cu - the non-GEMM pieces of the Swin backbones (SURVEY.md section 8 row a2; Swin-T/S/B/L, 7x7 or 12x12 windows), NHWC tokens.
//
// Reference: mmdet/models/backbones/swin_transformer.py - PatchEmbed :430-446, SwinTransformerBlock :199-256
// (norm1 -> zero pad to multiples of the window -> cyclic shift -> windows -> WindowAttention :122-154 -> reverse ->
// crop -> residual; norm2 -> MLP), PatchMerging :272-299, BasicLayer mask :371-390.  All Linear layers run on the
// tensor-core convolution kernel (dense_tc.cu) as 1x1 convolutions; here are LayerNorm (optionally scattering into
// the zero-padded window grid), the window attention itself (shift, relative-position bias and the -100 region mask
// are index arithmetic - no roll / partition / reverse copies), the 4x4 patch gather, the 2x2 merge gather and the
// stride-2 subsample that max_pool2d(kernel 1, stride 2) is (necks/fpn.py:163-165).
//
// Every kernel exists for both activation formats of the tensor-core engines: bf16 [.., C] and the f16x3 "split" format
// fp16 [.., 2, C] (per token C hi values, then C lo values, x = hi + lo); the arithmetic in between is fp32 either way.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/orp_b200_swin.h"
#include "act.cuh"
#include "common.cuh"

namespace orp {
namespace {

// one warp per token; out may be a padded grid [B,Hp,Wp,C] (rows beyond H,W pre-zeroed by the caller)
template <bool SPLIT, int kLnChunks>
__global__ void __launch_bounds__(256)
layernorm_kernel(const typename Act<SPLIT>::T *__restrict__ x, int B, int H, int W, int C, const float *__restrict__ gamma,
                 const float *__restrict__ beta, float eps, int Hp, int Wp, int G, typename Act<SPLIT>::T *__restrict__ y)
{
    // a group of G lanes (a power of two, G * kLnChunks >= C / 8) per token, 32 / G tokens per warp; a lane owns the 16-byte chunks
    // (8 channels) g, g + G, ... of its token: vector loads and stores, all lanes busy (C = 96: 4 lanes x 3 chunks, 8 tokens per warp)
    const int lane = threadIdx.x & 31, g = lane & (G - 1);
    const int tpw = 32 / G;                                                    // tokens per warp
    const long long tok = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * tpw + lane / G;
    const long long ntok = (long long)B * H * W;
    const bool live = tok < ntok;
    float v[kLnChunks][8];                         // 3 chunks per lane up to C = 768 (every block norm of Swin-T: few registers, high occupancy), 6 up to the 1536-wide PatchMerging norm, 12 up to 3072 (Swin-B / L)
    const int chunks = C >> 3;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kLnChunks; ++i) {
        const int ch = g + i * G;
        if (live && ch < chunks) {
            Act<SPLIT>::ld8(x, tok, C, ch * 8, v[i]);
#pragma unroll
            for (int j = 0; j < 8; ++j) s += v[i][j];
        }
    }
    for (int o = G >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < kLnChunks; ++i) {
        if (live && g + i * G < chunks) {
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; q += d * d; }
        }
    }
    for (int o = G >> 1; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if (!live) return;
    const float rstd = rsqrtf(q / (float)C + eps);
    const int b = (int)(tok / ((long long)H * W)), hw = (int)(tok - (long long)b * H * W);
    const int h = hw / W, w = hw - h * W;
    const long long otok = ((long long)b * Hp + h) * Wp + w;
#pragma unroll
    for (int i = 0; i < kLnChunks; ++i) {
        const int ch = g + i * G;
        if (ch < chunks) {
            const float4 g0 = *reinterpret_cast<const float4 *>(gamma + ch * 8), g1 = *reinterpret_cast<const float4 *>(gamma + ch * 8 + 4);
            const float4 b0 = *reinterpret_cast<const float4 *>(beta + ch * 8), b1 = *reinterpret_cast<const float4 *>(beta + ch * 8 + 4);
            const float ga[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, be[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            float o8[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) o8[j] = (v[i][j] - mean) * rstd * ga[j] + be[j];
            Act<SPLIT>::st8(y, otok, C, ch * 8, o8);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Window attention on the tensor cores (warp-level mma.sync m16n8k16, fp32 accumulation), one template over the window side
// WIN (7: orp_window_attention_*, 12: orp_window_attention12_*).  One block per (window, head), one warp per 16 query rows:
// the window's WIN^2 tokens are staged as kRows = 16 * ceil(WIN^2 / 16) rows (49 -> 64 in four warps; 144 = 9 x 16 in nine warps,
// no padded rows).  Q, K, V are staged as the 16-bit planes they are stored in (fp16 hi / lo in split mode, bf16 otherwise) - no
// conversion; S = Q K^T and O = P V are evaluated with the same three-term products as the convolutions (lo x hi, hi x lo, hi x hi),
// the probabilities P are split into a (hi, lo) pair in registers (both modes), bias + region mask + softmax run on the
// accumulator fragments in fp32.
// qkv: [B,Hp,Wp,3C] (q | k | v, each heads x 32), out: [B,H,W,C] at the ORIGINAL (unshifted, uncropped-away) positions.
// ---------------------------------------------------------------------------------------------
constexpr int kHd = 32;
constexpr int kAS = 40;            // shared-memory row pitch in 16-bit elements (80 B: conflict-free ldmatrix rows)

template <int WIN>
struct WinShape {
    static constexpr int kTok = WIN * WIN;                 // tokens per window
    static constexpr int kKSteps = (kTok + 15) / 16;       // 16-key steps of O = P V; also the warps (one 16-row query tile each)
    static constexpr int kRows = 16 * kKSteps;             // staged rows of q, k and v; rows kTok.. are zero
    static constexpr int kThreads = 32 * kKSteps;
    static constexpr int kKeyTiles = (kTok + 7) / 8;       // 8-key tiles of S = Q K^T that hold a key (7 of 8 / 18 of 18)
    static constexpr int kSpan = 2 * WIN - 1;              // relative offsets per axis
    static constexpr int kBias = kSpan * kSpan;            // rows of the relative-position bias table (169 / 529)
    // q, k, v, each [planes][kRows][kAS] 16-bit: 30 KiB for w7 in split mode, 67.5 KiB for w12 (dynamic, opted in beyond 48 KiB)
    static constexpr int smem_bytes(bool split) { return 3 * (split ? 2 : 1) * kRows * kAS * 2; }
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void *p)
{
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const void *p)
{
    const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
template <bool SPLIT>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    if (SPLIT)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// (x, y) -> packed 16-bit pair of the engine's format and the packed remainder pair
template <bool SPLIT>
__device__ __forceinline__ void split_pair(float x, float y, uint32_t &hi, uint32_t &lo)
{
    if (SPLIT) {
        const __half2 h = __floats2half2_rn(x, y);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(x - hf.x, y - hf.y);
        hi = *reinterpret_cast<const uint32_t *>(&h); lo = *reinterpret_cast<const uint32_t *>(&l);
    } else {
        const __nv_bfloat162 h = __floats2bfloat162_rn(x, y);
        const float2 hf = __bfloat1622float2(h);
        const __nv_bfloat162 l = __floats2bfloat162_rn(x - hf.x, y - hf.y);
        hi = *reinterpret_cast<const uint32_t *>(&h); lo = *reinterpret_cast<const uint32_t *>(&l);
    }
}

template <bool SPLIT, int WIN>
__global__ void __launch_bounds__(WinShape<WIN>::kThreads)
window_attention_mma_kernel(const typename Act<SPLIT>::T *__restrict__ qkv, int B, int H, int W, int Hp, int Wp, int C, int heads,
                            int shift, const float *__restrict__ bias_table /* [(2 WIN - 1)^2, heads] */, float scale,
                            typename Act<SPLIT>::T *__restrict__ out)
{
    typedef WinShape<WIN> WS;
    constexpr int kTok = WS::kTok, kRows = WS::kRows, kThreads = WS::kThreads, kSpan = WS::kSpan;
    constexpr int NP = SPLIT ? 2 : 1;                      // 16-bit planes per value
    extern __shared__ uint4 s_attn_qkv[];                  // q | k | v, each [NP][kRows][kAS]
    typedef uint16_t Tile[kRows][kAS];
    Tile *sq = reinterpret_cast<Tile *>(s_attn_qkv), *sk = sq + NP, *sv = sk + NP;
    __shared__ int s_src[kRows], s_reg[kRows], s_col[kRows];
    __shared__ float s_bias[WS::kBias];
    const int nww = Wp / WIN, nwh = Hp / WIN;
    const int head = blockIdx.y;
    const int wid = blockIdx.x % (nwh * nww), b = blockIdx.x / (nwh * nww);
    const int wy = wid / nww, wx = wid - wy * nww;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < kRows) {
        int src = 0, reg = 0;
        // relative position index (:107-118) = (ty - jy + WIN - 1) * kSpan + (tx - jx + WIN - 1) = [ty * kSpan + tx + (WIN - 1) (kSpan + 1)]
        // - [jy * kSpan + jx]: one table entry per token, the softmax loop subtracts
        const int tq = tid < kTok ? tid : kTok - 1;
        s_col[tid] = (tq / WIN) * kSpan + (tq % WIN);
        if (tid < kTok) {
            const int ty = tid / WIN, tx = tid - ty * WIN;
            const int ys = wy * WIN + ty, xs = wx * WIN + tx;                   // coordinates in the shifted frame
            int yo = ys + shift, xo = xs + shift;                                // roll(x, -shift): shifted[y] = x[(y + shift) % Hp]
            if (yo >= Hp) yo -= Hp;
            if (xo >= Wp) xo -= Wp;
            src = (b * Hp + yo) * Wp + xo;
            // BasicLayer mask regions (:376-387): slices (0,-WIN), (-WIN,-shift), (-shift,None) of the shifted frame
            const int hr = ys < Hp - WIN ? 0 : (ys < Hp - shift ? 1 : 2);
            const int wr = xs < Wp - WIN ? 0 : (xs < Wp - shift ? 1 : 2);
            reg = shift > 0 ? hr * 3 + wr : 0;
        }
        s_src[tid] = src;
        s_reg[tid] = reg;
    }
    for (int i = tid; i < WS::kBias; i += kThreads) s_bias[i] = bias_table[i * heads + head];
    __syncthreads();
    // stage the 16-byte chunks of q | k | v (both planes); rows kTok..kRows-1 are zero
    {
        // thread -> (16-byte chunk c4, plane pl) fixed, rows j = jb + kPass * i, tensor q | k | v: simple addressing, all loads in
        // flight before the first store
        constexpr int kPass = kThreads / (4 * NP);           // rows covered by one pass of the block
        constexpr int kRowIt = kRows / kPass;
        static_assert(kRowIt * kPass == kRows, "staging passes must tile the rows");
        const int c4 = tid & 3, pl = (tid >> 2) % NP, jb = tid / (4 * NP);
        uint4 val[kRowIt][3];
#pragma unroll
        for (int i = 0; i < kRowIt; ++i) {
            const int j = jb + kPass * i;
            const uint16_t *src = reinterpret_cast<const uint16_t *>(qkv) + ((size_t)s_src[j] * NP + pl) * (size_t)(3 * C) + head * kHd + c4 * 8;
#pragma unroll
            for (int ten = 0; ten < 3; ++ten)
                val[i][ten] = j < kTok ? *reinterpret_cast<const uint4 *>(src + ten * C) : make_uint4(0u, 0u, 0u, 0u);
        }
#pragma unroll
        for (int i = 0; i < kRowIt; ++i) {
            const int j = jb + kPass * i;
            *reinterpret_cast<uint4 *>(&sq[pl][j][c4 * 8]) = val[i][0];
            *reinterpret_cast<uint4 *>(&sk[pl][j][c4 * 8]) = val[i][1];
            *reinterpret_cast<uint4 *>(&sv[pl][j][c4 * 8]) = val[i][2];
        }
    }
    __syncthreads();
    if (warp * 16 >= kTok) return;                         // (never: the warps cover rows 0..kRows-1, the last one holds token kTok-1)
    const int g = lane >> 2, t4 = lane & 3, m0 = warp * 16;

    // ---- S = Q K^T (accumulator fragment: [0],[1] = row g, cols 2 t4, +1; [2],[3] = row g + 8)
    uint32_t aq[NP][2][4];
#pragma unroll
    for (int pl = 0; pl < NP; ++pl)
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) ldsm_x4(aq[pl][ks], &sq[pl][m0 + (lane & 15)][ks * 16 + (lane >> 4) * 8]);
    float sc[2 * WS::kKSteps][4];
#pragma unroll
    for (int j = 0; j < WS::kKeyTiles; ++j) {
        sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
        uint32_t bk[NP][4];
#pragma unroll
        for (int pl = 0; pl < NP; ++pl) ldsm_x4(bk[pl], &sk[pl][8 * j + (lane & 7)][(lane >> 3) * 8]);
        if (SPLIT) {
            mma16816<SPLIT>(sc[j], aq[NP - 1][0], bk[0][0], bk[0][1]); mma16816<SPLIT>(sc[j], aq[NP - 1][1], bk[0][2], bk[0][3]);      // q_lo k_hi
            mma16816<SPLIT>(sc[j], aq[0][0], bk[NP - 1][0], bk[NP - 1][1]); mma16816<SPLIT>(sc[j], aq[0][1], bk[NP - 1][2], bk[NP - 1][3]);   // q_hi k_lo
        }
        mma16816<SPLIT>(sc[j], aq[0][0], bk[0][0], bk[0][1]); mma16816<SPLIT>(sc[j], aq[0][1], bk[0][2], bk[0][3]);
    }
    // ---- q * scale (:138), + relative position bias (:107-118, :141-144), + region mask (:388-389), softmax over the kTok keys
    const int r0 = m0 + g, r1 = r0 + 8;
    const int q0 = r0 < kTok ? r0 : kTok - 1, q1 = r1 < kTok ? r1 : kTok - 1;     // padded rows compute on a clamped query, never stored
    const int rp0 = s_col[q0] + (WIN - 1) * kSpan + (WIN - 1), rp1 = s_col[q1] + (WIN - 1) * kSpan + (WIN - 1);
    const int rg0 = s_reg[q0], rg1 = s_reg[q1];
    float mx0 = -3.0e38f, mx1 = -3.0e38f;
#pragma unroll
    for (int j = 0; j < WS::kKeyTiles; ++j) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int c = 8 * j + 2 * t4 + u;
            if (c < kTok) {
                const int cp = s_col[c], rc = s_reg[c];
                float a0 = fmaf(sc[j][u], scale, s_bias[rp0 - cp]);
                float a1 = fmaf(sc[j][2 + u], scale, s_bias[rp1 - cp]);
                if (rg0 != rc) a0 += -100.0f;
                if (rg1 != rc) a1 += -100.0f;
                sc[j][u] = a0; sc[j][2 + u] = a1;
                mx0 = fmaxf(mx0, a0); mx1 = fmaxf(mx1, a1);
            } else {
                sc[j][u] = -3.0e38f; sc[j][2 + u] = -3.0e38f;
            }
        }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float den0 = 0.f, den1 = 0.f;
#pragma unroll
    for (int j = 0; j < WS::kKeyTiles; ++j)
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const bool in = (8 * j + 2 * t4 + u) < kTok;
            const float e0 = in ? expf(sc[j][u] - mx0) : 0.f, e1 = in ? expf(sc[j][2 + u] - mx1) : 0.f;
            sc[j][u] = e0; sc[j][2 + u] = e1;
            den0 += e0; den1 += e1;
        }
    den0 += __shfl_xor_sync(0xffffffffu, den0, 1); den0 += __shfl_xor_sync(0xffffffffu, den0, 2);
    den1 += __shfl_xor_sync(0xffffffffu, den1, 1); den1 += __shfl_xor_sync(0xffffffffu, den1, 2);
    const float inv0 = 1.0f / den0, inv1 = 1.0f / den1;
#pragma unroll
    for (int j = WS::kKeyTiles; j < 2 * WS::kKSteps; ++j)   // key tiles past the window (w7: keys 56..63) do not exist
        sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;

    // ---- O = P V: the accumulator fragments of two neighbouring key tiles are the A fragment of one 16-key step
    float o[4][4];
#pragma unroll
    for (int jn = 0; jn < 4; ++jn) o[jn][0] = o[jn][1] = o[jn][2] = o[jn][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < WS::kKSteps; ++kk) {
        uint32_t ph[4], pl_[4];
        split_pair<SPLIT>(sc[2 * kk][0] * inv0, sc[2 * kk][1] * inv0, ph[0], pl_[0]);
        split_pair<SPLIT>(sc[2 * kk][2] * inv1, sc[2 * kk][3] * inv1, ph[1], pl_[1]);
        split_pair<SPLIT>(sc[2 * kk + 1][0] * inv0, sc[2 * kk + 1][1] * inv0, ph[2], pl_[2]);
        split_pair<SPLIT>(sc[2 * kk + 1][2] * inv1, sc[2 * kk + 1][3] * inv1, ph[3], pl_[3]);
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            uint32_t bv[NP][4];
#pragma unroll
            for (int pl = 0; pl < NP; ++pl)
                ldsm_x4_trans(bv[pl], &sv[pl][16 * kk + ((lane >> 3) & 1) * 8 + (lane & 7)][16 * np + (lane >> 4) * 8]);
            mma16816<SPLIT>(o[2 * np], pl_, bv[0][0], bv[0][1]); mma16816<SPLIT>(o[2 * np + 1], pl_, bv[0][2], bv[0][3]);              // p_lo v_hi
            if (SPLIT) { mma16816<SPLIT>(o[2 * np], ph, bv[NP - 1][0], bv[NP - 1][1]); mma16816<SPLIT>(o[2 * np + 1], ph, bv[NP - 1][2], bv[NP - 1][3]); }   // p_hi v_lo
            mma16816<SPLIT>(o[2 * np], ph, bv[0][0], bv[0][1]); mma16816<SPLIT>(o[2 * np + 1], ph, bv[0][2], bv[0][3]);
        }
    }
    // ---- window_reverse + roll(+shift) + crop: a token returns to its original position if that is inside H x W
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int r = half ? r1 : r0;
        if (r >= kTok) continue;
        const int src = s_src[r];
        const int xo = src % Wp, yo = (src / Wp) % Hp;
        if (yo >= H || xo >= W) continue;
        const long long otok = ((long long)b * H + yo) * W + xo;
        uint16_t *dst = reinterpret_cast<uint16_t *>(out) + (size_t)otok * NP * C + head * kHd + 2 * t4;
#pragma unroll
        for (int jn = 0; jn < 4; ++jn) {
            float x = o[jn][2 * half], y = o[jn][2 * half + 1];
            uint32_t hi, lo;
            if (SPLIT) { x = fminf(fmaxf(x, -65504.f), 65504.f); y = fminf(fmaxf(y, -65504.f), 65504.f); }
            split_pair<SPLIT>(x, y, hi, lo);
            *reinterpret_cast<uint32_t *>(dst + 8 * jn) = hi;
            if (SPLIT) *reinterpret_cast<uint32_t *>(dst + C + 8 * jn) = lo;
        }
    }
}

// PatchEmbed.proj input rows: NCHW fp32 image -> bf16 [B, ceil(H/4), ceil(W/4), 64], k = c*16 + kh*4 + kw (< 48), zero padded
template <bool SPLIT>
__global__ void __launch_bounds__(256)
patch_embed_rows_kernel(const float *__restrict__ img, int B, int H, int W, int Ho, int Wo, typename Act<SPLIT>::T *__restrict__ out)
{
    const long long total = (long long)B * Ho * Wo * 64;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i & 63);
        const long long pix = i >> 6;
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
        float v = 0.f;
        if (k < 48) {
            const int c = k >> 4, kh = (k >> 2) & 3, kw = k & 3;
            const int y = oh * 4 + kh, x = ow * 4 + kw;
            if (y < H && x < W) v = img[(((long long)b * 3 + c) * H + y) * W + x];      // F.pad with zeros (:432-436)
        }
        Act<SPLIT>::st(out, pix, 64, k, v);
    }
}

// the same rows straight from decoded uint8 HWC tiles: Normalize (mmdet/datasets/pipelines/transforms.py: to_rgb, (x - mean) / std as
// (x - mean) * (1 / std), two roundings like the eager expression) + ImageToTensor fused into the gather
// valid (int32 [B,2] = (h, w) per image, or null for the full extent): pixels at y >= h or x >= w are the Pad step after
// Normalize and contribute exactly 0.0
struct NormCfg { float mean[3], stdinv[3]; int to_rgb; };
template <bool SPLIT>
__global__ void __launch_bounds__(256)
patch_embed_rows_u8_kernel(const uint8_t *__restrict__ img, int B, int H, int W, int Ho, int Wo, NormCfg nc,
                           const int32_t *__restrict__ valid, typename Act<SPLIT>::T *__restrict__ out)
{
    const long long total = (long long)B * Ho * Wo * 64;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i & 63);
        const long long pix = i >> 6;
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
        float v = 0.f;
        if (k < 48) {
            const int c = k >> 4, kh = (k >> 2) & 3, kw = k & 3;
            const int y = oh * 4 + kh, x = ow * 4 + kw;
            const int vh = valid ? min(valid[2 * b], H) : H, vw = valid ? min(valid[2 * b + 1], W) : W;
            if (y < vh && x < vw) {
                const float raw = (float)img[(((long long)b * H + y) * W + x) * 3 + (nc.to_rgb ? 2 - c : c)];
                v = __fmul_rn(__fsub_rn(raw, nc.mean[c]), nc.stdinv[c]);
            }
        }
        Act<SPLIT>::st(out, pix, 64, k, v);
    }
}

// PatchMerging gather (:288-293): [B,H,W,C] -> [B,ceil(H/2),ceil(W/2),4C] = x(0::2,0::2) | x(1::2,0::2) | x(0::2,1::2) | x(1::2,1::2)
// (16-bit elements of either format; P = planes per token: 1 bf16, 2 split - the hi and lo planes are gathered alike)
__global__ void __launch_bounds__(256)
patch_merge_gather_kernel(const uint16_t *__restrict__ x, int B, int H, int W, int C, int P, int Ho, int Wo,
                          uint16_t *__restrict__ y)
{
    const int c8 = C / 8;
    const long long total = (long long)B * Ho * Wo * P * 4 * c8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cc = (int)(i % c8);
        const int part = (int)((i / c8) & 3);
        const int pl = (int)((i / (4LL * c8)) % P);
        const long long pix = i / (4LL * c8 * P);
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
        const int yy = oh * 2 + (part & 1), xx = ow * 2 + (part >> 1);
        uint4 v = make_uint4(0, 0, 0, 0);
        if (yy < H && xx < W) v = *reinterpret_cast<const uint4 *>(x + ((((long long)b * H + yy) * W + xx) * P + pl) * C + cc * 8);
        *reinterpret_cast<uint4 *>(y + (pix * P + pl) * (4LL * C) + (long long)part * C + cc * 8) = v;
    }
}

// max_pool2d(kernel_size=1, stride=2) == x[:, ::2, ::2, :]
__global__ void __launch_bounds__(256)
subsample2_kernel(const uint16_t *__restrict__ x, int B, int H, int W, int C /* 16-bit elements per token, planes included */, int Ho, int Wo,
                  uint16_t *__restrict__ y)
{
    const int c8 = C / 8;
    const long long total = (long long)B * Ho * Wo * c8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int cc = (int)(i % c8);
        const long long pix = i / c8;
        const int ow = (int)(pix % Wo), oh = (int)((pix / Wo) % Ho), b = (int)(pix / ((long long)Wo * Ho));
        reinterpret_cast<uint4 *>(y)[i] = *reinterpret_cast<const uint4 *>(x + (((long long)b * H + oh * 2) * W + ow * 2) * C + cc * 8);
    }
}

}  // namespace
}  // namespace orp

using namespace orp;

// WIDE: the 1536 < C <= 3072 PatchMerging norms of Swin-B / Swin-L (orp_layernorm_wide_*), 12 chunks per lane at G = 32
template <bool SPLIT, bool WIDE>
static int layernorm_impl(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps, int Hp, int Wp,
                          void *y, void *stream)
{
    if (WIDE) {
        if (!x || !y || !gamma || !beta || C <= 1536 || C > 3072 || (C & 7) || Hp < H || Wp < W)
            return fail(ORP_EINVAL, "layernorm_wide: C must be a multiple of 8, 1536 < C <= 3072");
    } else if (!x || !y || !gamma || !beta || C < 8 || C > 1536 || (C & 7) || Hp < H || Wp < W) {
        return fail(ORP_EINVAL, "layernorm: C must be a multiple of 8, <= 1536");
    }
    int rc = ensure_device();
    if (rc) return rc;
    const long long ntok = (long long)B * H * W;
    typedef typename Act<SPLIT>::T T;
    // lanes per token: the smallest power of two whose lanes hold the token in at most kLnChunks 16-byte chunks each - for Swin-T's
    // widths (96 / 192 / 384 / 768 -> 4 / 8 / 16 / 32 lanes x 3 chunks) no lane idles
    const int kLnChunks = WIDE ? 12 : (C <= 768 ? 3 : 6);
    int G = 1;
    while (G < 32 && G * kLnChunks < (C >> 3)) G <<= 1;
    const long long tok_per_block = 8LL * (32 / G);
    const unsigned nblk = (unsigned)((ntok + tok_per_block - 1) / tok_per_block);
    if (WIDE)
        layernorm_kernel<SPLIT, 12><<<nblk, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const T *>(x), B, H, W, C, gamma, beta, eps,
                                                                                         Hp, Wp, G, static_cast<T *>(y));
    else if (kLnChunks == 3)
        layernorm_kernel<SPLIT, 3><<<nblk, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const T *>(x), B, H, W, C, gamma, beta, eps,
                                                                                        Hp, Wp, G, static_cast<T *>(y));
    else
        layernorm_kernel<SPLIT, 6><<<nblk, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const T *>(x), B, H, W, C, gamma, beta, eps,
                                                                                        Hp, Wp, G, static_cast<T *>(y));
    ORP_LAUNCHED();
    return ORP_OK;
}
extern "C" int orp_layernorm_bf16(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps,
                                  int Hp, int Wp, void *y, void *stream)
{
    return layernorm_impl<false, false>(x, B, H, W, C, gamma, beta, eps, Hp, Wp, y, stream);
}
extern "C" int orp_layernorm_f16x3(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps,
                                   int Hp, int Wp, void *y, void *stream)
{
    return layernorm_impl<true, false>(x, B, H, W, C, gamma, beta, eps, Hp, Wp, y, stream);
}
extern "C" int orp_layernorm_wide_bf16(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps,
                                       int Hp, int Wp, void *y, void *stream)
{
    return layernorm_impl<false, true>(x, B, H, W, C, gamma, beta, eps, Hp, Wp, y, stream);
}
extern "C" int orp_layernorm_wide_f16x3(const void *x, int B, int H, int W, int C, const float *gamma, const float *beta, float eps,
                                        int Hp, int Wp, void *y, void *stream)
{
    return layernorm_impl<true, true>(x, B, H, W, C, gamma, beta, eps, Hp, Wp, y, stream);
}

template <bool SPLIT, int WIN>
static int window_attention_impl(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                 const float *bias_table, float scale, void *out, void *stream)
{
    if (!qkv || !out || !bias_table || heads * kHd != C || Hp % WIN || Wp % WIN || shift < 0 || shift >= WIN)
        return fail(ORP_EINVAL, WIN == 7 ? "window_attention: needs 7x7 windows, head_dim 32, padded grid"
                                         : "window_attention12: needs 12x12 windows, head_dim 32, padded grid");
    int rc = ensure_device();
    if (rc) return rc;
    typedef WinShape<WIN> WS;
    constexpr int smem = WS::smem_bytes(SPLIT);
    auto kern = window_attention_mma_kernel<SPLIT, WIN>;
    if (smem > 48 * 1024) {                      // opt in to more than 48 KiB of dynamic shared memory, once per device
        static int opted[64];
        int dev = 0;
        ORP_CUDA(cudaGetDevice(&dev));
        if (dev >= 64 || !__atomic_load_n(&opted[dev], __ATOMIC_ACQUIRE)) {
            ORP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            if (dev < 64) __atomic_store_n(&opted[dev], 1, __ATOMIC_RELEASE);
        }
    }
    dim3 grid(B * (Hp / WIN) * (Wp / WIN), heads);
    typedef typename Act<SPLIT>::T T;
    kern<<<grid, WS::kThreads, smem, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const T *>(qkv), B, H, W, Hp, Wp, C, heads, shift, bias_table, scale, static_cast<T *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}
extern "C" int orp_window_attention_bf16(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                         const float *bias_table, float scale, void *out, void *stream)
{
    return window_attention_impl<false, 7>(qkv, B, H, W, Hp, Wp, C, heads, shift, bias_table, scale, out, stream);
}
extern "C" int orp_window_attention_f16x3(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                          const float *bias_table, float scale, void *out, void *stream)
{
    return window_attention_impl<true, 7>(qkv, B, H, W, Hp, Wp, C, heads, shift, bias_table, scale, out, stream);
}
extern "C" int orp_window_attention12_bf16(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                           const float *bias_table, float scale, void *out, void *stream)
{
    return window_attention_impl<false, 12>(qkv, B, H, W, Hp, Wp, C, heads, shift, bias_table, scale, out, stream);
}
extern "C" int orp_window_attention12_f16x3(const void *qkv, int B, int H, int W, int Hp, int Wp, int C, int heads, int shift,
                                            const float *bias_table, float scale, void *out, void *stream)
{
    return window_attention_impl<true, 12>(qkv, B, H, W, Hp, Wp, C, heads, shift, bias_table, scale, out, stream);
}

template <bool SPLIT>
static int patch_embed_rows_impl(const float *img_nchw, int B, int H, int W, void *out, void *stream)
{
    if (!img_nchw || !out) return fail(ORP_EINVAL, "patch_embed_rows: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 3) / 4, Wo = (W + 3) / 4;
    patch_embed_rows_kernel<SPLIT><<<grid_for((long long)B * Ho * Wo * 64, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img_nchw, B, H, W, Ho, Wo, static_cast<typename Act<SPLIT>::T *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}
extern "C" int orp_patch_embed_rows_bf16(const float *img_nchw, int B, int H, int W, void *out, void *stream)
{
    return patch_embed_rows_impl<false>(img_nchw, B, H, W, out, stream);
}
extern "C" int orp_patch_embed_rows_f16x3(const float *img_nchw, int B, int H, int W, void *out, void *stream)
{
    return patch_embed_rows_impl<true>(img_nchw, B, H, W, out, stream);
}

template <bool SPLIT>
static int patch_embed_rows_u8_impl(const uint8_t *img_hwc, int B, int H, int W, const float *mean, const float *stdinv, int to_rgb,
                                    const int32_t *valid, void *out, void *stream)
{
    if (!img_hwc || !out || !mean || !stdinv) return fail(ORP_EINVAL, "patch_embed_rows_u8: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    NormCfg nc;
    for (int c = 0; c < 3; ++c) { nc.mean[c] = mean[c]; nc.stdinv[c] = stdinv[c]; }
    nc.to_rgb = to_rgb ? 1 : 0;
    const int Ho = (H + 3) / 4, Wo = (W + 3) / 4;
    patch_embed_rows_u8_kernel<SPLIT><<<grid_for((long long)B * Ho * Wo * 64, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        img_hwc, B, H, W, Ho, Wo, nc, valid, static_cast<typename Act<SPLIT>::T *>(out));
    ORP_LAUNCHED();
    return ORP_OK;
}
extern "C" int orp_patch_embed_rows_u8_bf16(const uint8_t *img_hwc, int B, int H, int W, const float *mean, const float *stdinv,
                                            int to_rgb, void *out, void *stream)
{
    return patch_embed_rows_u8_impl<false>(img_hwc, B, H, W, mean, stdinv, to_rgb, nullptr, out, stream);
}
extern "C" int orp_patch_embed_rows_u8_f16x3(const uint8_t *img_hwc, int B, int H, int W, const float *mean, const float *stdinv,
                                             int to_rgb, void *out, void *stream)
{
    return patch_embed_rows_u8_impl<true>(img_hwc, B, H, W, mean, stdinv, to_rgb, nullptr, out, stream);
}
extern "C" int orp_patch_embed_rows_u8_padded_bf16(const uint8_t *img_hwc, int B, int H, int W, const float *mean,
                                                   const float *stdinv, int to_rgb, const int32_t *valid_hw, void *out, void *stream)
{
    if (!valid_hw) return fail(ORP_EINVAL, "patch_embed_rows_u8_padded_bf16: valid_hw is required");
    return patch_embed_rows_u8_impl<false>(img_hwc, B, H, W, mean, stdinv, to_rgb, valid_hw, out, stream);
}
extern "C" int orp_patch_embed_rows_u8_padded_f16x3(const uint8_t *img_hwc, int B, int H, int W, const float *mean,
                                                    const float *stdinv, int to_rgb, const int32_t *valid_hw, void *out, void *stream)
{
    if (!valid_hw) return fail(ORP_EINVAL, "patch_embed_rows_u8_padded_f16x3: valid_hw is required");
    return patch_embed_rows_u8_impl<true>(img_hwc, B, H, W, mean, stdinv, to_rgb, valid_hw, out, stream);
}

static int patch_merge_gather_impl(const void *x, int B, int H, int W, int C, int P, void *y, void *stream)
{
    if (!x || !y || C % 8) return fail(ORP_EINVAL, "patch_merge_gather: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    patch_merge_gather_kernel<<<grid_for((long long)B * Ho * Wo * P * 4 * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint16_t *>(x), B, H, W, C, P, Ho, Wo, static_cast<uint16_t *>(y));
    ORP_LAUNCHED();
    return ORP_OK;
}
extern "C" int orp_patch_merge_gather_bf16(const void *x, int B, int H, int W, int C, void *y, void *stream)
{
    return patch_merge_gather_impl(x, B, H, W, C, 1, y, stream);
}
extern "C" int orp_patch_merge_gather_f16x3(const void *x, int B, int H, int W, int C, void *y, void *stream)
{
    return patch_merge_gather_impl(x, B, H, W, C, 2, y, stream);
}

static int subsample2_impl(const void *x, int B, int H, int W, int Cel, void *y, void *stream)
{
    if (!x || !y || Cel % 8) return fail(ORP_EINVAL, "subsample2: bad arguments");
    int rc = ensure_device();
    if (rc) return rc;
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    subsample2_kernel<<<grid_for((long long)B * Ho * Wo * (Cel / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint16_t *>(x), B, H, W, Cel, Ho, Wo, static_cast<uint16_t *>(y));
    ORP_LAUNCHED();
    return ORP_OK;
}
extern "C" int orp_subsample2_bf16(const void *x, int B, int H, int W, int C, void *y, void *stream)
{
    return subsample2_impl(x, B, H, W, C, y, stream);
}
extern "C" int orp_subsample2_f16x3(const void *x, int B, int H, int W, int C, void *y, void *stream)
{
    return subsample2_impl(x, B, H, W, 2 * C, y, stream);       // a split token is 2 C contiguous 16-bit elements
}
