// dense_tc.cu - tensor-core (wgmma / TMA / mbarrier) implicit-GEMM convolution for sm_90a (H100), NHWC bf16.
//
// Replaces the cuDNN convolutions of the reference's backbone / FPN / head towers
// (mmdet/models/backbones/resnet.py:203-239,495-506; necks/fpn.py:138-178;
// anchor_heads/orientedreppoints_head.py:153-168) and, in its gathered-operand variant, the deformable
// im2col + SGEMM of mmdet/ops/dcn/src/deform_conv_cuda.cpp:152-260.
//
// GEMM view: D[M = 128 output pixels, N = BN output channels] += A[M, K] * B[N, K]^T with
// K = taps x Cin walked in 64-channel blocks.  One persistent CTA per SM, warp-specialised:
//   warps 0-7   two consumer warpgroups.  Warpgroup g issues wgmma.mma_async m64nBNk16 x 4 per stage for the
//               output rows [64 g, 64 g + 64), accumulating fp32 in registers, and releases the stage once the
//               MMAs that read it have retired.  After the last K block the same warps run the epilogue: the
//               accumulator is staged in shared memory 64 columns at a time (fp32, one row per pixel), then
//               bias / residual / ReLU and bf16, split-fp16 or fp32 NHWC stores.  (The deformable f16x3 variant that
//               computes N-tile pairs, 256 columns wide, finishes straight from its register fragments: frag_epilogue.)
//   warp 8      TMA producer (plain variant): the A tile of one (tap, channel block) is ONE box {64 ch, BW, BH, BI}
//               of the NHWC activation (tensor-map element strides = conv stride; out-of-bounds
//               coordinates are zero-filled by the TMA unit = the convolution's zero padding), landing in
//               shared memory as 128 rows x 128 B with the 128-byte swizzle - exactly the canonical
//               K-major operand layout of wgmma; the B tile is a 2-D box of the [Cout, K] weights.
//   warps 8-15  (deformable variant only) A-operand producers: per output pixel and tap the 4-corner
//               bilinear sample of the reference (deform_conv_cuda_kernel.cu:84-115) is computed in
//               fp32 from bf16 features and written to shared memory in the same swizzled layout; their first
//               thread also issues the TMA loads of the B tiles.  In f16x3 with 16-bit outputs (the detector's head)
//               a CTA computes two adjacent 128-wide N tiles as one 256-wide tile (plan field n_pair), so every sample
//               is taken once: setmaxnreg moves registers from these warps to the consumers, whose fragment is then
//               64 x 256 fp32.
// Several "problems" (the five FPN levels, which share the head weights) are served by ONE launch.
//
// Two operand modes share the kernel.  bf16: activations / weights rounded to bf16, one MMA per K step.
// f16x3 ("split"): every fp32 value is carried as an fp16 pair x = hi + lo (22 significand bits, activations
// stored [N,H,W,2,C]: hi channels then lo channels per pixel) and every product is evaluated as
// hi*hi + lo*hi + hi*lo with three MMAs into the same fp32 accumulator (the dropped lo*lo term is 2^-22
// relative) - fp32-faithful arithmetic at 1/3 of the tensor-pipe rate; this is the parity mode.  The K loop
// simply runs three "terms" per (tap, channel block); weights are stored [Cout][tap][channel block][2][64] = (hi, lo).
// For layers with BN <= 128 output channels per tile the terms are concatenated along N instead of K ("ncat"): per K
// step  x_hi * w_hi  goes to accumulator columns [0, BN), and  x_hi * w_lo  then  x_lo * w_hi  to [BN, 2 BN) - the
// x_hi / x_lo tiles of a (tap, channel block) are loaded once, and the small cross terms own an accumulator (their sum
// never meets the large main sum before the epilogue adds the two in fp32).
// Operand type and walk are template parameters (SPLIT, WALK): every K block is one straight-line MMA sequence, which
// ptxas needs to keep the MMAs in flight.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"

namespace orp {
namespace {

constexpr int kMaxProb = 5;
constexpr int kStagesMax = 6;
constexpr int kBM = 128;
constexpr int kBK = 64;                       // bf16 elements per K block = 128 bytes = one swizzle row
constexpr int kABytes = kBM * kBK * 2;        // 16 KiB

// division by a runtime constant as multiply-high + shift (Granlund-Montgomery); exact for 0 <= n < 2^31
struct FastDiv {
    uint32_t mul, shr, d;
    __host__ void set(uint32_t div)
    {
        d = div;
        uint32_t l = 0;
        while ((1ull << l) < div) ++l;
        shr = l;
        mul = (uint32_t)(((1ull << 32) * ((1ull << l) - div)) / div + 1);
    }
    __device__ __forceinline__ uint32_t div(uint32_t n) const { return (__umulhi(n, mul) + n) >> shr; }   // n < 2^31: no overflow
    __device__ __forceinline__ void divmod(uint32_t n, uint32_t &q, uint32_t &r) const { q = div(n); r = n - q * d; }
};

struct Problem {
    int N, H, W, Ho, Wo;
    FastDiv fd_tw, fd_th;                     // / tiles_w, / tiles_h
    int BW, BH, BI;                           // tile box: BW*BH*BI == 128 output pixels (powers of two)
    int lbw, lbh;                             // log2(BW), log2(BH)
    int tiles_w, tiles_h, tiles_i, tile_start;
    void *out;                                // bf16 / split-fp16 or fp32 NHWC [N,Ho,Wo,(2,)Cout]
    const __nv_bfloat16 *res;                 // optional residual, same layout as the 16-bit output
    const float *res32;                       // optional fp32 residual (head: refine += init)
    const __nv_bfloat16 *x;                   // activation base (deformable variant; fp16 pairs in split mode)
    const float *offset;                      // deformable: [N,Ho,Wo,2*taps] fp32
    const float *mask;                        // deformable, optional DCNv2 modulation: [N,Ho,Wo,taps] fp32
    double *gn_stats;                         // optional [N, 32, 2] (sum, sum of squares) of the output, GroupNorm(32)
};

struct alignas(64) TcParams {
    CUtensorMap tmA[kMaxProb];
    CUtensorMap tmB;
    CUtensorMap tmOut[kMaxProb];              // bf16 output tensors, box {64 ch, BW, BH, BI} (TMA-store epilogue)
    CUtensorMap tmRes[kMaxProb];              // bf16 residual tensors, same boxes
    CUtensorMap tmI;                          // 64 x 64 bf16 identity (residual add on the tensor core)
    Problem prob[kMaxProb];
    int tma_epi, epi_bufs;                    // TMA epilogue on/off; output staging buffers (1 or 2)
    int epi_merge;                            // split mode, memory-bound layers: hi and lo tiles of a 64-column group leave in ONE pass
    int ncat;                                 // split mode, BN <= 128: terms concatenated along N (see the kernel header)
    int ksplit;                               // split-K over the taps (launches with fewer tiles than SMs): partial sums meet in an fp32 buffer
    FastDiv fd_ks;                            // / ksplit
    long long ks_stride;                      // elements between the partial-sum slabs of consecutive K splits
    int b_resident;                           // short-K layers: the whole weight slab of this CTA's N tile stays in shared memory
    int res_mma;                              // residual added by the tensor core: extra K blocks  R[128x64] * I[64x64]
    int gn_fused;                             // GroupNorm statistics accumulated in the TMA epilogue (Cout == 256)
    int dcat;                                 // deformable split mode: one stage = sampled x_hi | x_lo | w_hi | w_lo of a K block
    int split;                                // f16x3 mode: fp16 (hi, lo) operand pairs, three MMA terms per K block
    float oscale;                             // epilogue multiplier 2^-s undoing the power-of-two weight scale (split mode)
    unsigned int *ovf;                        // split mode: count of outputs beyond the fp16 range (saturated)
    int nprob, num_m_tiles, n_tiles_n, num_tiles;
    FastDiv fd_ntn;                           // / n_tiles_n
    int KH, KW, Cin, cin_blocks, stride, pad, Cout, relu;
    int s2d_stem;                             // conv1 in space-to-depth form (host bookkeeping: 147 useful K of 256)
    const float *bias;
};

// ----------------------------------------------------------------------------------------------- PTX
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ bool elect_one()
{
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "elect.sync _|P1, %1;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t"
        "}" : "=r"(pred) : "r"(0xffffffffu));
    return pred != 0;
}
__device__ __forceinline__ void tma_load_4d(void *smem, const CUtensorMap *tm, uint64_t *bar, int c0, int c1, int c2, int c3)
{
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_5d(void *smem, const CUtensorMap *tm, uint64_t *bar, int c0, int c1, int c2, int c3, int c4)
{
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *smem, const CUtensorMap *tm, uint64_t *bar, int c0, int c1)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem)), "l"(tm), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// wgmma matrix descriptor, K-major with the 128-byte swizzle: start address >> 4, LBO = 1 (ignored), SBO = 1024 B >> 4
// (eight 128-byte rows), layout type 1 = SWIZZLE_128B in bits 62-63.  Operand tiles start on 1024-byte boundaries.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ uint4 lds128(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const uint4 &v)
{
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
template <int ID, int N>
__device__ __forceinline__ void named_bar()
{
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory");
}
// 32 consecutive fp32 columns of one staged accumulator row (conflict-free: 16-byte loads, row pitch 68 words)
__device__ __forceinline__ void acc_ld32(uint32_t addr, uint32_t (&r)[32])
{
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const uint4 v = lds128(addr + (uint32_t)j * 16u);
        r[4 * j] = v.x; r[4 * j + 1] = v.y; r[4 * j + 2] = v.z; r[4 * j + 3] = v.w;
    }
}

// two fp32 lanes, each rounded once (sm_90 has no packed fp32 FMA / add)
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 fadd2_rn(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

// One split-mode deformable sample of 8 channels: the (hi, lo) fp16 rows u[c][0 / 1] of the four corners c blended with
// the corner weights (wv in fp32; wh the same four as fp16), formed in fp32 and split again into x_hi and x_lo.
__device__ __forceinline__ void split_sample(const uint4 (&u)[4][2], float4 wv, uint2 wh, uint32_t (&hi)[4], uint32_t (&lo)[4])
{
    const float2 wc[4] = {make_float2(wv.x, wv.x), make_float2(wv.y, wv.y), make_float2(wv.z, wv.z), make_float2(wv.w, wv.w)};
    const __half2 wl[4] = {__low2half2(*reinterpret_cast<const __half2 *>(&wh.x)), __high2half2(*reinterpret_cast<const __half2 *>(&wh.x)),
                           __low2half2(*reinterpret_cast<const __half2 *>(&wh.y)), __high2half2(*reinterpret_cast<const __half2 *>(&wh.y))};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        // hi halves: fp32, two channels per packed FMA; lo halves (<= 2^-11 of the value): blended in half2 arithmetic with
        // fp16 weights - an error of 2^-11 on a 2^-11 term
        float2 acc = make_float2(0.f, 0.f);
        __half2 accl = __float2half2_rn(0.f);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const uint32_t uh = reinterpret_cast<const uint32_t *>(&u[c][0])[k];
            const uint32_t ul = reinterpret_cast<const uint32_t *>(&u[c][1])[k];
            acc = ffma2_rn(wc[c], __half22float2(*reinterpret_cast<const __half2 *>(&uh)), acc);
            accl = __hfma2(wl[c], *reinterpret_cast<const __half2 *>(&ul), accl);
        }
        acc = fadd2_rn(acc, __half22float2(accl));
        const __half2 h2 = __floats2half2_rn(acc.x, acc.y);
        const float2 hf = __half22float2(h2);
        const float2 rem = fadd2_rn(acc, make_float2(-hf.x, -hf.y));
        const __half2 l2 = __floats2half2_rn(rem.x, rem.y);
        hi[k] = *reinterpret_cast<const uint32_t *>(&h2);
        lo[k] = *reinterpret_cast<const uint32_t *>(&l2);
    }
}

// epilogue activation: 0 none, 1 ReLU, 2 exact (erf) GELU as nn.GELU (swin_transformer.py:24-29)
__device__ __forceinline__ float act_fn(float v, int act)
{
    if (act == 1) return fmaxf(v, 0.f);
    if (act == 2) return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
    return v;
}

struct Ring {
    int stage = 0;
    uint32_t phase = 0;
    int n;
    __device__ explicit Ring(int n_) : n(n_) {}
    __device__ void next() { if (++stage == n) { stage = 0; phase ^= 1; } }
};

// Walk of the main-loop K blocks of one tile: (tap, term, channel block).
//   bf16:                     tap-major, one term.
//   split, TMA operands:      the cross terms (1: x_lo * w_hi, 2: x_hi * w_lo) of ALL taps first, then the main terms
//                             (0: x_hi * w_hi).  The tensor core truncates its fp32 accumulator on every K step (measured:
//                             error grows linearly with the step count, 6e-6 of max at 432 steps); while only the 2^-11
//                             times smaller cross terms have been added the accumulator's ulp - hence that loss - is 2^-11
//                             times smaller too, so the loss of a tile is that of K/16 steps instead of 3K/16.
//   split, deformable:        tap-major, one stage per (tap, channel block) carrying both halves of both operands (dcat): the
//                             producers sample once and hand the K block over once - with one stage per term they could
//                             only start the next gather after the THIRD stage of a block had been freed, which exposed
//                             two thirds of the gather time.
struct KIter {
    int tap, term, cb = 0, phase = 0;
    int tap0, taps, cbn, mode;                             // taps [tap0, taps); mode 0: one stage per K block, 1: split TMA (a stage per term)
    __device__ KIter(int taps_, int cbn_, int mode_, int tap0_ = 0) : tap0(tap0_), taps(taps_), cbn(cbn_), mode(mode_)
    {
        tap = tap0;
        term = (mode == 1) ? 1 : 0;
    }
    __device__ void next()
    {
        if (mode == 0) { if (++cb == cbn) { cb = 0; ++tap; } }
        else if (phase == 0) {
            if (++cb == cbn) { cb = 0; if (++term == 3) { term = 1; if (++tap == taps) { tap = tap0; term = 0; phase = 1; } } }
        } else { if (++cb == cbn) { cb = 0; ++tap; } }
    }
};

__device__ __forceinline__ int ksplit_of(const TcParams &P, int tile)
{
    if (P.ksplit <= 1) return 0;
    uint32_t q, r;
    P.fd_ks.divmod((uint32_t)tile, q, r);
    return (int)r;
}

__device__ __forceinline__ void decode_tile(const TcParams &P, int tile, int &pi, int &wb, int &hb, int &ib, int &nt)
{
    uint32_t mt_u, nt_u;
    if (P.ksplit > 1) tile = (int)P.fd_ks.div((uint32_t)tile);          // tile = (m tile, n tile, k split), k split fastest
    P.fd_ntn.divmod((uint32_t)tile, mt_u, nt_u);
    nt = (int)nt_u;
    const int mt = (int)mt_u;
    pi = 0;
#pragma unroll
    for (int k = 1; k < kMaxProb; ++k)
        if (k < P.nprob && mt >= P.prob[k].tile_start) pi = k;
    const Problem &pr = P.prob[pi];
    const int local = mt - pr.tile_start;
    uint32_t rest, wb_u, ib_u, hb_u;
    pr.fd_tw.divmod((uint32_t)local, rest, wb_u);
    pr.fd_th.divmod(rest, ib_u, hb_u);
    wb = (int)wb_u; hb = (int)hb_u; ib = (int)ib_u;
}

// 64 x 64 bf16 identity, the B operand that adds a residual tile into the accumulator
struct IdentBlock { unsigned short v[64 * 64]; };
constexpr IdentBlock make_ident()
{
    IdentBlock b{};
    for (int i = 0; i < 64; ++i) b.v[i * 64 + i] = 0x3F80;   // bf16 1.0
    return b;
}
__device__ IdentBlock g_ident = make_ident();
// split mode: 2^s * identity in fp16 for s = 0..15 (the weights of a layer carry a power-of-two scale 2^s that
// the epilogue removes, so the residual has to enter the accumulator scaled alike)
struct IdentBlocks16 { unsigned short v[16][64 * 64]; };
constexpr IdentBlocks16 make_ident16()
{
    IdentBlocks16 b{};
    for (int s = 0; s < 16; ++s)
        for (int i = 0; i < 64; ++i) b.v[s][i * 64 + i] = (unsigned short)((15 + s) << 10);   // fp16 2^s
    return b;
}
__device__ IdentBlocks16 g_ident16 = make_ident16();
__device__ unsigned int g_f16_overflow = 0;

// ----------------------------------------------------------------------------------------------- kernel
constexpr int kConsumers = 256;                    // two consumer warpgroups: MMA, then epilogue (warps 0-7)
constexpr int kDP = 256;                           // deformable A-operand producer threads (warps 8 .. 8 + kDP/32 - 1)
constexpr int kDItems = 1024 / kDP;                // (pixel row, 8-channel chunk) items of one 128 x 64 A block per thread
constexpr int kDRound = kDItems / 2;               // items gathered together (two rounds per K block)
constexpr int kAccPitch = 68;                      // words per staged accumulator row: 64 columns + 4 (conflict-free 16-byte reads)
constexpr int kAccBytes = 128 * kAccPitch * 4;     // one 64-column pass of the 128 x BN accumulator, fp32 (34 KiB)

// bytes of one main-loop stage: the A tile (x_hi | x_lo when a stage carries both halves: ncat, dcat) and, unless the weight
// slab of the CTA's N tile is resident, the B tile (w_hi | w_lo likewise)
__host__ __device__ constexpr int stage_bytes(int BN, bool cat, bool b_resident)
{
    return cat ? (b_resident ? 2 * kABytes : 2 * kABytes + 2 * BN * kBK * 2) : (b_resident ? kABytes : kABytes + BN * kBK * 2);
}
// The deformable f16x3 variant of N-tile pairs (256 accumulator columns) runs its epilogue straight from the fragments: its two 96 KiB stages
// leave no room for the staged accumulator pass.  Every other variant stages the accumulator (stage_acc).
__host__ __device__ constexpr bool frag_epilogue(int BN, bool deform) { return deform && BN == 256; }
// dynamic shared memory of a launch: 1 KiB alignment slack, the staged accumulator pass (unless frag_epi), `stages`
// main-loop stages and `extra` bytes (identity block, resident weight slab, output staging)
constexpr int dyn_smem_bytes(int stage_b, int stages, int extra, bool frag_epi)
{
    return 1024 + (frag_epi ? 0 : kAccBytes) + stages * stage_b + extra;
}

// Columns [64 pass, 64 pass + 64) of this thread's accumulator fragment -> the staged rows (ncat: main + cross columns,
// added here in fp32 with round-to-nearest).  The pass loop is unrolled with a compile-time index so that the fragment
// stays in registers.  row0 / col0: the fragment's first row and column (wgmma.cuh).
template <int BN, int R>
__device__ __forceinline__ void stage_acc(const float (&acc)[R], int pass, bool ncat, float *s_acc, int row0, int col0)
{
    constexpr int kGroups = (BN < 64 ? BN : 64) / 8;         // 8-column groups per pass
#pragma unroll
    for (int p = 0; p < (BN + 63) / 64; ++p) {
        if (p != pass) continue;
#pragma unroll
        for (int i = 0; i < kGroups; ++i) {
            const int g = p * 8 + i;
            float2 a = make_float2(acc[4 * g], acc[4 * g + 1]), b = make_float2(acc[4 * g + 2], acc[4 * g + 3]);
            if constexpr (R >= BN) {
                if (ncat) {                                   // cross columns: BN further on, BN / 2 registers further
                    a.x += acc[BN / 2 + 4 * g]; a.y += acc[BN / 2 + 4 * g + 1];
                    b.x += acc[BN / 2 + 4 * g + 2]; b.y += acc[BN / 2 + 4 * g + 3];
                }
            }
            *reinterpret_cast<float2 *>(s_acc + row0 * kAccPitch + i * 8 + col0) = a;
            *reinterpret_cast<float2 *>(s_acc + (row0 + 8) * kAccPitch + i * 8 + col0) = b;
        }
    }
}

// Main-loop walk of an instantiation (the MMA sequence of a K block is fixed at compile time: ptxas serialises wgmma
// instructions that sit behind run-time branches).
constexpr int kWalkK = 0;        // one stage per K block and term: bf16, or f16x3 with a stage per term (KIter mode 1)
constexpr int kWalkNcat = 1;     // f16x3, terms concatenated along N: BN <= 128, TMA epilogue, no residual
constexpr int kWalkDcat = 2;     // deformable f16x3: one stage carries x_hi | x_lo | w_hi | w_lo of a K block
constexpr int kWalkKRes = 3;     // kWalkK, then the residual K blocks (res_mma: residual tile x identity into the accumulator)

// accumulator columns [64 G, 64 G + 64) += A * B[rows 64 G ..]^T for G = 0 .. NG - 1: one width-64 MMA per column group
// (the B rows of group G start 64 rows = 8 KiB further, 512 in the descriptor's address field)
template <int NG, bool BF16, int R, int G = 0>
__device__ __forceinline__ void wgmma_cols64(float (&acc)[R], uint64_t da, uint64_t db, uint32_t accumulate)
{
    wgmma_n<64, BF16>(acc_view<32 * G, 32>(acc), da, db + (uint64_t)(G * 512), accumulate);
    if constexpr (G + 1 < NG) wgmma_cols64<NG, BF16, R, G + 1>(acc, da, db, accumulate);
}

// accumulator (+)= A * B^T over BN columns (dcat walk): one MMA, or at BN = 256 two of 128 columns each - an m64n256 MMA
// names 128 accumulator registers, all that the 512-thread launch of the deformable variant gives a thread (ptxas allots
// an instruction's operands against the launch's count, not the setmaxnreg budget).  The B rows of the second half start
// 128 rows = 16 KiB further, 1024 in the descriptor's address field.  Every column sees the MMA sequence of the 128-wide plan.
template <int BN, bool BF16>
__device__ __forceinline__ void wgmma_dcat(float (&acc)[BN / 2], uint64_t da, uint64_t db, uint32_t accumulate)
{
    if constexpr (BN == 256) {
        wgmma_n<128, BF16>(acc_view<0, 64>(acc), da, db, accumulate);
        wgmma_n<128, BF16>(acc_view<64, 64>(acc), da, db + (uint64_t)1024, accumulate);
    } else {
        wgmma_n<BN, BF16>(acc, da, db, accumulate);
    }
}

// Register budgets of the plain variant (384 threads launched with 168 registers each = 64 512 of the SM's 65 536): the
// TMA producer's warpgroup gives registers back, the two consumer warpgroups take them for the accumulator and the
// epilogue.  2 * 128 * 232 + 128 * 40 = 64 512.
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
// ... and of the wide deformable variant (512 threads launched with 128 registers each): the two gathering warpgroups
// give registers to the two consumer warpgroups, whose 64 x 256 fp32 fragment alone takes 128.  96 keep two items' corner
// loads in flight per producer thread, as in the 128-wide variant.  2 * 128 * 160 + 2 * 128 * 96 = 65 536.
constexpr int kWideConsumerRegs = 160;
constexpr int kWideProducerRegs = 96;

// BN: accumulator width (32..256).  OUT_F32: fp32 output (head predictions) instead of bf16.  DEFORM: A operand produced
// by the warps from 8 on (bilinear gather) instead of TMA.  SPLIT: f16x3 (fp16 operand pairs) instead of bf16.  WALK:
// kWalkK / kWalkKRes / kWalkNcat / kWalkDcat.
template <int BN, bool OUT_F32, bool DEFORM, bool SPLIT, int WALK>
__global__ void __launch_bounds__(DEFORM ? kConsumers + kDP : kConsumers + 128, 1)
conv_tc_kernel(const __grid_constant__ TcParams P, int stages)
{
    static_assert(WALK != kWalkNcat || (SPLIT && !DEFORM && !OUT_F32 && BN >= 64 && BN <= 128), "ncat: f16x3 TMA-epilogue layers, BN 64..128");
    static_assert(!DEFORM || (WALK == kWalkDcat) == SPLIT, "deformable: dcat exactly in f16x3");
    static_assert(DEFORM || WALK != kWalkDcat, "dcat is the deformable walk");
    static_assert(WALK != kWalkKRes || (!DEFORM && !OUT_F32 && BN >= 64), "residual K blocks: TMA-epilogue layers");
    constexpr bool kBF16 = !SPLIT;                     // operand type of every MMA
    constexpr int kWTerms = SPLIT ? 2 : 1;             // weight K blocks per (tap, channel block): hi, lo
    constexpr bool kCat = WALK == kWalkNcat || WALK == kWalkDcat;             // a stage holds both halves of both operands
    constexpr int kKMode = (SPLIT && !kCat) ? 1 : 0;   // KIter mode: a stage per term
    static_assert(kConsumers + 128 == 384 && 2 * 128 * kConsumerRegs + 128 * kProducerRegs <= 65536, "register split");
    constexpr bool kFragEpi = frag_epilogue(BN, DEFORM);
    static_assert(!kFragEpi || (SPLIT && !OUT_F32), "fragment epilogue: deformable f16x3 with a TMA epilogue");
    static_assert(kConsumers == 256 && kDP == 256 && 2 * 128 * kWideConsumerRegs + 2 * 128 * kWideProducerRegs <= 65536,
                  "register split (wide deformable)");
    // warp roles.  0-7: consumer warpgroups (wgmma main loop, then epilogue).  plain: 8 TMA producer (9-11 idle).
    // deformable: 8-15 A-operand producers, their thread 0 also loads the B tiles.
    constexpr int kEpiThreads = kConsumers;
    constexpr int kWG = 2;                             // epilogue warps per 32-row quarter (one per 32-column half)
    // accumulator columns per thread group: the ncat layout (BN <= 128) keeps main | cross columns side by side
    constexpr int kAccN = (WALK == kWalkNcat) ? 2 * BN : BN;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // dynamic: [staged accumulator pass][identity][resident B][stages: A 16K | B BN*128] then the output staging tile
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    float *s_acc = reinterpret_cast<float *>(smem);
    if constexpr (!kFragEpi) smem += kAccBytes;
    constexpr int kBBytes = BN * kBK * 2;
    // b_resident: [B slab: kblocks x kBBytes] then A-only stages; otherwise every stage carries A | B
    const int kStageBytes = stage_bytes(BN, kCat, P.b_resident);
    const int kblocks_all = P.KH * P.KW * P.cin_blocks * kWTerms;   // weight K blocks (hi and lo halves in split mode)
    uint8_t *ident = smem;                             // [8 KiB] identity block when res_mma
    if (P.res_mma) smem += 8192;
    uint8_t *bres = smem;
    if (P.b_resident) smem += (size_t)kblocks_all * kBBytes;
    constexpr int HC = BN < 64 ? BN : 64;              // columns staged per epilogue pass
    constexpr int kPitch = HC * 2 + 16;                // bytes per staged row (+16: conflict-free 16-byte accesses)
    uint8_t *stage_out = smem + (size_t)stages * kStageBytes;
    __shared__ uint64_t bars[2 * kStagesMax];
    __shared__ __align__(16) float s_bias[256];
    __shared__ uint64_t bres_bar;                // resident weight slab landed
    uint64_t *full = bars;                       // [stages]  TMA bytes landed (+ producer arrivals when DEFORM)
    uint64_t *empty = bars + kStagesMax;         // [stages]  both consumer warpgroups' MMAs finished reading the stage

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == kConsumers / 32 && elect_one()) {
        if (!DEFORM) {
#pragma unroll 1
            for (int p = 0; p < P.nprob; ++p)
                asm volatile("prefetch.tensormap [%0];" ::"l"(&P.tmA[p]) : "memory");
        }
        asm volatile("prefetch.tensormap [%0];" ::"l"(&P.tmB) : "memory");
    }
    if (warp == 0) {
        if (elect_one()) {
            for (int s = 0; s < stages; ++s) {
                mbar_init(&full[s], DEFORM ? 1 + kDP / 32 : 1);                          // TMA expect_tx arrival (+ one arrival per producer warp)
                mbar_init(&empty[s], kConsumers / 128);                                 // one arrival per consumer warpgroup
            }
            mbar_init(&bres_bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncwarp();
    }
    __syncthreads();
    const int taps_per = (P.KH * P.KW) / (P.ksplit > 1 ? P.ksplit : 1);              // taps of one K split
    const int kblocks = taps_per * P.cin_blocks * (kKMode ? 3 : 1);     // main-loop K blocks (stages) per tile
    // Programmatic dependent launch: the next kernel in the stream may start its CTAs (barrier init, descriptor
    // prefetch - the code above) on SMs this grid has already left; nothing above touches global memory,
    // and everything below (loads AND stores) comes after the wait for the preceding grid to complete and flush.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");

    if (warp < kConsumers / 32) {
        // ===================================================== consumers: main loop
        if constexpr (!DEFORM) setmaxnreg_inc<kConsumerRegs>();
        if constexpr (kFragEpi) setmaxnreg_inc<kWideConsumerRegs>();
        const int cw = warp >> 2;                          // consumer warpgroup: accumulator rows [64 cw, 64 cw + 64)
        const uint32_t a_off = (uint32_t)cw * 8192u;       // its 64 rows of a 128-row A tile (64 x 128 B)
        const bool leader = (threadIdx.x & 127) == 0;
        float acc[kAccN / 2];
        Ring r(stages);
        // epilogue geometry: thread -> staged row rrow = q * 32 + lane, 32-column half wg of every 64-column pass
        const int q = warp & 3, wg = warp >> 2;
        const int et = threadIdx.x, nthr = kEpiThreads;
        const int bar_a = 1, bar_b = 3;                    // named barriers of the consumers; 2 = deformable producers
        const int ch0 = wg, chs = kWG;
        const int frow = cw * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);   // fragment's first row / column
        const uint32_t s_acc_u = smem_u32(s_acc);
        auto bar_sync = [](int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); };
        int ob = 0;                                        // staging ring position (TMA epilogue)
        int bias_nt = -1;                                  // N tile whose bias slice is staged in s_bias
        if ((P.b_resident || P.res_mma) && (int)blockIdx.x < P.num_tiles) mbar_wait(&bres_bar, 0);
        for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
            int res_groups = 0;
            if constexpr (WALK == kWalkKRes) {
                const int nt = tile - (int)P.fd_ntn.div((uint32_t)tile) * P.n_tiles_n;
                for (int g = 0; g < BN / 64 && nt * BN + g * 64 < P.Cout; ++g) ++res_groups;
            }
            const int tap_lo = ksplit_of(P, tile) * taps_per;
            KIter it(tap_lo + taps_per, P.cin_blocks, kKMode, tap_lo);   // same walk as the producer
            // A stage is released once the MMAs reading it have retired: with one commit group in flight, the stage
            // before the current one.
            int held = -1;
            auto release = [&](int next) {
                if (held >= 0 && leader) mbar_arrive(&empty[held]);
                held = next;
            };
            for (int kb = 0; kb < kblocks; ++kb, it.next()) {
                if constexpr (kFragEpi) {
                    // The wide deformable variant is bound by its gather and has two stages only: the previous K block's
                    // MMAs retire and free their stage BEFORE the wait for the next one, so that the producers, which
                    // write a stage as they sample it, find it free when they start on it.
                    wgmma_wait<0>();
                    release(-1);
                }
                mbar_wait(&full[r.stage], r.phase);
                const uint32_t sa = smem_u32(smem + (size_t)r.stage * kStageBytes);
                const uint64_t da = make_desc_sw128(sa + a_off);
                const int slab = (it.tap * P.cin_blocks + it.cb) * kWTerms + (it.term == 2 ? 1 : 0);
                wgmma_fence();
                if constexpr (WALK == kWalkNcat) {
                    // [w_hi | w_lo] are adjacent in the stage (and in the resident slab).  x_hi * w_hi goes to the main
                    // columns, x_hi * w_lo then x_lo * w_hi to the cross columns.  All three MMAs have the width BN:
                    // successive MMAs into the same accumulator registers are ordered without a wait only when their
                    // shapes are equal.
                    const uint32_t sb = P.b_resident ? smem_u32(bres + (size_t)slab * kBBytes) : sa + 2 * kABytes;
                    const uint64_t dl = make_desc_sw128(sa + kABytes + a_off);
                    const uint64_t dbh = make_desc_sw128(sb), dbl = make_desc_sw128(sb + kBBytes);
#pragma unroll
                    for (int k = 0; k < kBK / 16; ++k) {
                        const uint32_t first = (kb | k) ? 1u : 0u;
                        wgmma_n<BN, kBF16>(acc_view<0, BN / 2>(acc), da + (uint64_t)(k * 2), dbh + (uint64_t)(k * 2), first);        // x_hi * w_hi
                        wgmma_n<BN, kBF16>(acc_view<BN / 2, BN / 2>(acc), da + (uint64_t)(k * 2), dbl + (uint64_t)(k * 2), first);   // x_hi * w_lo
                        wgmma_n<BN, kBF16>(acc_view<BN / 2, BN / 2>(acc), dl + (uint64_t)(k * 2), dbh + (uint64_t)(k * 2), 1u);      // x_lo * w_hi
                    }
                } else if constexpr (WALK == kWalkDcat) {
                    const uint64_t dl = make_desc_sw128(sa + kABytes + a_off);
                    const uint64_t dbh = make_desc_sw128(sa + 2 * kABytes), dbl = make_desc_sw128(sa + 2 * kABytes + kBBytes);
#pragma unroll
                    for (int k = 0; k < kBK / 16; ++k) {
                        wgmma_dcat<BN, kBF16>(acc, dl + (uint64_t)(k * 2), dbh + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);   // x_lo * w_hi
                        wgmma_dcat<BN, kBF16>(acc, da + (uint64_t)(k * 2), dbl + (uint64_t)(k * 2), 1u);                   // x_hi * w_lo
                        wgmma_dcat<BN, kBF16>(acc, da + (uint64_t)(k * 2), dbh + (uint64_t)(k * 2), 1u);                   // x_hi * w_hi
                    }
                } else {
                    const uint64_t db = make_desc_sw128(P.b_resident ? smem_u32(bres + (size_t)slab * kBBytes) : sa + kABytes);
#pragma unroll
                    for (int k = 0; k < kBK / 16; ++k) {
                        if constexpr (WALK == kWalkKRes)     // the shape of the residual blocks' MMAs (see there)
                            wgmma_cols64<BN / 64, kBF16>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
                        else
                            wgmma_n<BN, kBF16>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) ? 1u : 0u);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
                release(r.stage);
                r.next();
            }
            if constexpr (WALK == kWalkKRes) {
                // residual K blocks: accumulator columns [64 G, 64 G + 64) += residual tile * (scaled) identity, a block per
                // group G and term, all MMAs of width 64 like the main loop's in this walk (with width-BN main-loop MMAs on
                // the same registers ptxas serialises every MMA of the kernel, C7511).  The main loop's last group retires
                // first, unconditionally: the epilogue would wait for it anyway.
                wgmma_wait<0>();
                release(-1);
                auto res_group = [&](auto gc) {
                    constexpr int G = decltype(gc)::value;
                    if (G >= res_groups) return;
#pragma unroll 1
                    for (int t = 0; t < kWTerms; ++t) {
                        mbar_wait(&full[r.stage], r.phase);
                        const uint64_t da = make_desc_sw128(smem_u32(smem + (size_t)r.stage * kStageBytes) + a_off);
                        const uint64_t db = make_desc_sw128(smem_u32(ident));
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < kBK / 16; ++k)
                            wgmma_n<64, kBF16>(acc_view<32 * G, 32>(acc), da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), 1u);
                        wgmma_commit();
                        wgmma_wait<1>();
                        release(r.stage);
                        r.next();
                    }
                };
                res_group(std::integral_constant<int, 0>{});
                if constexpr (BN >= 128) res_group(std::integral_constant<int, 1>{});
                if constexpr (BN >= 256) {
                    res_group(std::integral_constant<int, 2>{});
                    res_group(std::integral_constant<int, 3>{});
                }
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            release(-1);

            // ===================================================== epilogue
            int pi, wb, hb, ib, nt;
            decode_tile(P, tile, pi, wb, hb, ib, nt);
            const Problem &pr = P.prob[pi];
            const int rrow = q * 32 + lane;
            auto row_pixel = [&](int r, size_t &pix) -> bool {
                const int iw = r & (pr.BW - 1), ih = (r >> pr.lbw) & (pr.BH - 1), ii = r >> (pr.lbw + pr.lbh);
                const int w = wb * pr.BW + iw, h = hb * pr.BH + ih, n = ib * pr.BI + ii;
                pix = ((size_t)n * pr.Ho + h) * pr.Wo + w;
                return (w < pr.Wo) && (h < pr.Ho) && (n < pr.N);
            };
            size_t pix;
            const bool valid = row_pixel(rrow, pix);
            if constexpr (kFragEpi) {
                // Epilogue from the fragments (no staged accumulator pass): every consumer thread finishes its own values
                // with the arithmetic of the staged TMA epilogue below, in the same order, and writes them to the
                // 128-byte-swizzled staging tile 4 bytes (a column pair) at a time - the 8 rows x 4 column pairs of a
                // warp's store fall in 32 distinct banks.  A hi and a lo pass per 64 columns, each leaving with one TMA store.
                const uint32_t obuf_u = smem_u32(stage_out);             // [epi_bufs][16 KiB]
                const bool io = (et == 0);
                if (nt != bias_nt) {
                    bar_sync(bar_a, nthr);                               // previous tile's bias reads are done
                    for (int c = et; c < BN; c += nthr) s_bias[c] = (P.bias && nt * BN + c < P.Cout) ? P.bias[nt * BN + c] : 0.f;
                    bias_nt = nt;
                }
                size_t pix_r[2];
                const bool valid_r[2] = {row_pixel(frow, pix_r[0]), row_pixel(frow + 8, pix_r[1])};
                // per fragment row (frow, frow + 8) and 32-column half of the passes: the staged epilogue's per-thread maxima
                float amax[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
                for (int pass = 0; pass < 2 * (BN / 64); ++pass) {
                    const int half = pass >> 1, oterm = pass & 1;
                    if (io) {
                        if (P.epi_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    bar_sync(bar_a, nthr);                               // staging buffer `ob` is free, bias staged
                    const uint32_t obase = obuf_u + (uint32_t)ob * 16384u;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int g = half * 8 + i;                      // 8-column group of the fragment
                        const float2 bv = *reinterpret_cast<const float2 *>(&s_bias[g * 8 + fcol]);
#pragma unroll
                        for (int hr = 0; hr < 2; ++hr) {
                            const int row = frow + 8 * hr;
                            float f0 = acc[4 * g + 2 * hr], f1 = acc[4 * g + 2 * hr + 1];
                            f0 *= P.oscale; f1 *= P.oscale;              // exact: power of two
                            f0 += bv.x; f1 += bv.y;
                            if (P.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }     // (n_pair plans have no GELU)
                            if (oterm == 0) amax[hr][i >> 2] = fmaxf(fmaxf(amax[hr][i >> 2], fabsf(f0)), fabsf(f1));
                            const __half2 h2 = __floats2half2_rn(f0, f1);
                            uint32_t v = *reinterpret_cast<const uint32_t *>(&h2);
                            if (oterm) {
                                const float2 hf = __half22float2(h2);
                                const __half2 l2 = __floats2half2_rn(f0 - hf.x, f1 - hf.y);
                                v = *reinterpret_cast<const uint32_t *>(&l2);
                            }
                            const uint32_t at = obase + (uint32_t)row * 128u + ((uint32_t)(i ^ (row & 7)) << 4) + (uint32_t)fcol * 2u;
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(at), "r"(v) : "memory");
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    bar_sync(bar_b, nthr);                               // staging written by all
                    if (io) {
                        asm volatile(
                            "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                            ::"l"(&P.tmOut[pi]), "r"(obase), "r"(nt * BN + half * 64), "r"(oterm),
                              "r"(wb * pr.BW), "r"(hb * pr.BH), "r"(ib * pr.BI) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                    if (++ob == P.epi_bufs) ob = 0;
                }
                // the overflow count of the staged epilogue: one per output pixel and 32-column half with a value beyond the
                // fp16 range (the four lanes of a fragment row hold its columns)
#pragma unroll
                for (int hr = 0; hr < 2; ++hr)
#pragma unroll
                    for (int hc = 0; hc < 2; ++hc) {
                        float m = amax[hr][hc];
                        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
                        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                        if ((lane & 3) == 0 && valid_r[hr] && m > 65504.f) atomicAdd(P.ovf, 1u);
                    }
            } else if (OUT_F32) {
                // fp32 outputs (head predictions, split-K partial sums): straight from the staged rows
#pragma unroll 1
                for (int pass = 0; pass < BN / HC; ++pass) {
                bar_sync(bar_a, nthr);                               // the previous pass's reads of the staged rows are done
                stage_acc<BN>(acc, pass, false, s_acc, frow, fcol);
                bar_sync(bar_a, nthr);
#pragma unroll 1
                for (int ch = wg; ch < HC / 32; ch += kWG) {
                    uint32_t v[32];
                    acc_ld32(s_acc_u + (uint32_t)(rrow * kAccPitch + ch * 32) * 4u, v);
                    const int c0 = nt * BN + pass * HC + ch * 32;
                    if (valid && c0 < P.Cout) {
                        float *op = reinterpret_cast<float *>(pr.out) + pix * P.Cout + c0;
                        const float *rp = pr.res32 ? pr.res32 + pix * P.Cout + c0 : nullptr;
                        if (P.ksplit > 1) {
                            // split-K: this tile holds the sum over its taps only and writes it to its own slab of the fp32
                            // workspace; the finishing kernel adds the slabs in a fixed order (bit-reproducible, unlike atomics)
                            // and applies bias / activation / the hi-lo split
                            float *sp = op + (long long)ksplit_of(P, tile) * P.ks_stride;
                            for (int j = 0; j < 32; ++j) {
                                if (c0 + j >= P.Cout) break;
                                sp[j] = __uint_as_float(v[j]) * P.oscale;
                            }
                        } else
                        for (int j = 0; j < 32; ++j) {
                            if (c0 + j >= P.Cout) break;
                            float f = __uint_as_float(v[j]) * P.oscale;
                            if (P.bias) f += P.bias[c0 + j];
                            if (pr.res && !P.split) f += __bfloat162float(pr.res[pix * P.Cout + c0 + j]);
                            if (rp) f += rp[j];
                            f = act_fn(f, P.relu);
                            op[j] = f;
                        }
                    }
                }
                }
            } else if (P.tma_epi) {
                // bf16 outputs through the TMA unit, in 64-channel passes: results go to a 128-byte-swizzled staging
                // tile and leave with cp.async.bulk.tensor (coalescing and partial-tile clipping by hardware).  A
                // residual is already in the accumulator (added by the tensor core, see the main loop).
                // Each of the two warps of a row quarter owns one 32-column half of the pass.
                const uint32_t slot = P.epi_merge ? 32768u : 16384u;     // a staging slot: one 16 KiB tile (hi | lo when merged)
                const uint32_t obuf_u = smem_u32(stage_out);             // [epi_bufs][slot]
                const uint32_t bias_u = smem_u32(s_bias);
                const bool io = (et == 0);
                constexpr int kPasses = BN / 64;
                // split mode: a hi pass and a lo pass per 64 columns (compute-bound layers: one 16 KiB staging tile), or both
                // halves in one pass (memory-bound layers: half the staged-row reads, barriers and fp32 work per output value)
                const int oterms = (P.split && !P.epi_merge) ? 2 : 1;
                if (nt != bias_nt) {                                     // bias slice changes only with the N tile
                    bar_sync(bar_a, nthr);                               // previous tile's bias reads are done
                    for (int c = et; c < BN; c += nthr) s_bias[c] = (P.bias && nt * BN + c < P.Cout) ? P.bias[nt * BN + c] : 0.f;
                    bias_nt = nt;
                }
                float amax = 0.f;
#pragma unroll 1
                for (int pass = 0; pass < kPasses * oterms; ++pass) {
                    const int half = oterms == 2 ? (pass >> 1) : pass, oterm = oterms == 2 ? (pass & 1) : 0;
                    if (io) {
                        if (P.epi_bufs == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
                        else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    }
                    bar_sync(bar_a, nthr);                               // staging buffer `ob` is free, bias staged, staged rows read
                    if (oterm == 0) {                                    // the lo pass of a half reads the rows its hi pass staged
                        stage_acc<BN>(acc, half, P.ncat != 0, s_acc, frow, fcol);
                        bar_sync(bar_a, nthr);
                    }
                    float gn_s = 0.f, gn_q = 0.f;
                    const uint32_t orow = obuf_u + (uint32_t)ob * slot + (uint32_t)rrow * 128u;
#pragma unroll 1
                    for (int ch = ch0; ch < 2; ch += chs) {
                        const uint32_t arow = s_acc_u + (uint32_t)(rrow * kAccPitch + ch * 32) * 4u;
#pragma unroll
                        for (int j4 = 0; j4 < 4; ++j4) {
                            const int c16 = ch * 4 + j4;                  // 16-byte chunk inside the 128-byte row
                            const uint32_t sw = (uint32_t)(c16 ^ (rrow & 7)) << 4;
                            const uint4 a0 = lds128(arow + (uint32_t)j4 * 32u), a1 = lds128(arow + (uint32_t)j4 * 32u + 16u);
                            const float f0[8] = {__uint_as_float(a0.x), __uint_as_float(a0.y), __uint_as_float(a0.z), __uint_as_float(a0.w),
                                                 __uint_as_float(a1.x), __uint_as_float(a1.y), __uint_as_float(a1.z), __uint_as_float(a1.w)};
                            float f[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) f[j] = f0[j];
                            const uint32_t bb = bias_u + (uint32_t)(half * 64 + ch * 32 + j4 * 8) * 4u;
                            const uint4 b0 = lds128(bb), b1 = lds128(bb + 16u);
                            if (P.split) {
#pragma unroll
                                for (int j = 0; j < 8; ++j) f[j] *= P.oscale;      // exact: power of two
                            }
                            f[0] += __uint_as_float(b0.x); f[1] += __uint_as_float(b0.y);
                            f[2] += __uint_as_float(b0.z); f[3] += __uint_as_float(b0.w);
                            f[4] += __uint_as_float(b1.x); f[5] += __uint_as_float(b1.y);
                            f[6] += __uint_as_float(b1.z); f[7] += __uint_as_float(b1.w);
                            if (P.relu == 2) {
#pragma unroll
                                for (int j = 0; j < 8; ++j) f[j] = act_fn(f[j], 2);
                            }
                            uint32_t pk[4];
                            if (P.split) {
                                // x = hi + lo with hi = fp16(x), lo = fp16(x - hi): 22 significand bits.  Values beyond the fp16
                                // range become inf / nan in the output AND are counted (P.ovf): never silent.
#pragma unroll
                                for (int j = 0; j < 8; ++j) {
                                    if (P.relu == 1) f[j] = fmaxf(f[j], 0.f);
                                    if (oterm == 0) amax = fmaxf(amax, fabsf(f[j]));
                                }
                                uint32_t pl[4];
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                    const __half2 h2 = __floats2half2_rn(f[2 * k], f[2 * k + 1]);
                                    pk[k] = *reinterpret_cast<const uint32_t *>(&h2);
                                    if (P.epi_merge || oterm) {
                                        const float2 hf = __half22float2(h2);
                                        const __half2 l2 = __floats2half2_rn(f[2 * k] - hf.x, f[2 * k + 1] - hf.y);
                                        pl[k] = *reinterpret_cast<const uint32_t *>(&l2);
                                    }
                                }
                                if (P.epi_merge) sts128(orow + 16384u + sw, make_uint4(pl[0], pl[1], pl[2], pl[3]));
                                else if (oterm) { pk[0] = pl[0]; pk[1] = pl[1]; pk[2] = pl[2]; pk[3] = pl[3]; }
                            } else {
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                    __nv_bfloat162 b2 = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
                                    // ReLU after rounding: rounding is monotone and keeps the sign, so the result is the same
                                    if (P.relu == 1) b2 = __hmax2(b2, __floats2bfloat162_rn(0.f, 0.f));
                                    pk[k] = *reinterpret_cast<uint32_t *>(&b2);
                                }
                            }
                            sts128(orow + sw, make_uint4(pk[0], pk[1], pk[2], pk[3]));
                            if (P.gn_fused && oterm == 0) {
                                // one 16-byte chunk = 8 channels = one GroupNorm group (Cout 256 / 32 groups)
                                float gs = 0.f, gq = 0.f;
                                if (valid) {
#pragma unroll
                                    for (int j = 0; j < 8; ++j) { gs += f[j]; gq = fmaf(f[j], f[j], gq); }
                                }
#pragma unroll
                                for (int o = 16; o > 0; o >>= 1) {
                                    gs += __shfl_xor_sync(0xffffffffu, gs, o);
                                    gq += __shfl_xor_sync(0xffffffffu, gq, o);
                                }
                                if (lane == c16) { gn_s = gs; gn_q = gq; }      // lane g keeps group g of this pass
                            }
                        }
                    }
                    if (P.gn_fused && oterm == 0 && lane < 8 && (chs == 1 || (lane >> 2) == wg)) {
                        // the 32 rows of a warp belong to one image (host guarantees BW*BH >= 32)
                        const int n_img = ib * pr.BI + ((q * 32) >> (pr.lbw + pr.lbh));
                        if (n_img < pr.N) {
                            double *st = pr.gn_stats + ((size_t)n_img * 32 + (size_t)(nt * BN + half * 64) / 8 + lane) * 2;
                            atomicAdd(st, (double)gn_s);
                            atomicAdd(st + 1, (double)gn_q);
                        }
                    }
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                    bar_sync(bar_b, nthr);                               // staging written by all
                    if (io) {
                        asm volatile(
                            "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                            ::"l"(&P.tmOut[pi]), "r"(obuf_u + (uint32_t)ob * slot), "r"(nt * BN + half * 64), "r"(oterm),
                              "r"(wb * pr.BW), "r"(hb * pr.BH), "r"(ib * pr.BI) : "memory");
                        if (P.epi_merge)
                            asm volatile(
                                "cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                                ::"l"(&P.tmOut[pi]), "r"(obuf_u + (uint32_t)ob * slot + 16384u), "r"(nt * BN + half * 64), "r"(1),
                                  "r"(wb * pr.BW), "r"(hb * pr.BH), "r"(ib * pr.BI) : "memory");
                        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                    }
                    if (++ob == P.epi_bufs) ob = 0;
                }
                if (P.split && valid && amax > 65504.f) atomicAdd(P.ovf, 1u);
            } else {
                // bf16 outputs: residual tile prefetched into shared memory with coalesced cp.async while the
                // MMA is still running, results written back to the same staging tile, then stored coalesced
                const bool vec_ok = (P.Cout & 7) == 0;
                named_bar<1, kEpiThreads>();
                for (int c = et; c < BN; c += kEpiThreads) s_bias[c] = (P.bias && nt * BN + c < P.Cout) ? P.bias[nt * BN + c] : 0.f;
                named_bar<1, kEpiThreads>();
#pragma unroll 1
                for (int half = 0; half < BN / HC; ++half) {
                    const int cbase = nt * BN + half * HC;           // first output channel of this pass
                    constexpr int kChunksPerRow = HC / 8;            // 16-byte chunks per staged row
                    if (pr.res && vec_ok) {
                        for (int c = et; c < 128 * kChunksPerRow; c += kEpiThreads) {
                            const int r = c / kChunksPerRow, k16 = c - r * kChunksPerRow;
                            size_t rp;
                            const bool ok = row_pixel(r, rp) && (cbase + k16 * 8 < P.Cout);
                            const uint32_t dst = smem_u32(stage_out + (size_t)r * kPitch + k16 * 16);
                            if (ok) {
                                const __nv_bfloat16 *src = pr.res + rp * P.Cout + cbase + k16 * 8;
                                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
                            }
                        }
                        asm volatile("cp.async.commit_group;" ::: "memory");
                    }
                    if (pr.res && vec_ok) asm volatile("cp.async.wait_group 0;" ::: "memory");
                    stage_acc<BN>(acc, half, false, s_acc, frow, fcol);
                    named_bar<1, kEpiThreads>();                         // residual tile and accumulator pass staged
#pragma unroll 1
                    for (int ch = wg; ch < HC / 32; ch += kWG) {
                        uint32_t v[32];
                        acc_ld32(s_acc_u + (uint32_t)(rrow * kAccPitch + ch * 32) * 4u, v);
                        const int c0 = cbase + ch * 32;
                        uint4 *sp = reinterpret_cast<uint4 *>(stage_out + (size_t)rrow * kPitch + ch * 64);
#pragma unroll
                        for (int j4 = 0; j4 < 4; ++j4) {
                            float f[8];
#pragma unroll
                            for (int j = 0; j < 8; ++j) f[j] = __uint_as_float(v[j4 * 8 + j]);
                            {
                                const float4 b0 = *reinterpret_cast<const float4 *>(&s_bias[half * HC + ch * 32 + j4 * 8]);
                                const float4 b1 = *reinterpret_cast<const float4 *>(&s_bias[half * HC + ch * 32 + j4 * 8 + 4]);
                                f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                                f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                            }
                            if (pr.res && !vec_ok && valid) {
                                for (int j = 0; j < 8; ++j)
                                    if (c0 + j4 * 8 + j < P.Cout) f[j] += __bfloat162float(pr.res[pix * P.Cout + c0 + j4 * 8 + j]);
                            }
                            if (pr.res && vec_ok && valid) {
                                const uint4 u = sp[j4];
                                const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                                for (int k = 0; k < 4; ++k) {
                                    const float2 r2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&uu[k]));
                                    f[2 * k] += r2.x;
                                    f[2 * k + 1] += r2.y;
                                }
                            }
                            if (P.relu) {
#pragma unroll
                                for (int j = 0; j < 8; ++j) f[j] = act_fn(f[j], P.relu);
                            }
                            uint32_t pk[4];
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                __nv_bfloat162 b2 = __floats2bfloat162_rn(f[2 * k], f[2 * k + 1]);
                                pk[k] = *reinterpret_cast<uint32_t *>(&b2);
                            }
                            sp[j4] = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                        }
                    }
                    named_bar<1, kEpiThreads>();
                    // coalesced copy-out: 16 threads cover one 256-byte row segment
                    for (int c = et; c < 128 * kChunksPerRow; c += kEpiThreads) {
                        const int r = c / kChunksPerRow, k16 = c - r * kChunksPerRow;
                        size_t rp;
                        if (row_pixel(r, rp) && (cbase + k16 * 8 < P.Cout)) {
                            const uint4 u = *reinterpret_cast<const uint4 *>(stage_out + (size_t)r * kPitch + k16 * 16);
                            __nv_bfloat16 *op = reinterpret_cast<__nv_bfloat16 *>(pr.out) + rp * P.Cout + cbase + k16 * 8;
                            if (vec_ok) {
                                *reinterpret_cast<uint4 *>(op) = u;
                            } else {
                                const __nv_bfloat16 *e8 = reinterpret_cast<const __nv_bfloat16 *>(&u);
                                for (int j = 0; j < 8; ++j) if (cbase + k16 * 8 + j < P.Cout) op[j] = e8[j];
                            }
                        }
                    }
                    named_bar<1, kEpiThreads>();
                }
            }
        }
        if (P.tma_epi && et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // stores drained before exit
    } else if (!DEFORM) {
        // ===================================================== TMA producer
        setmaxnreg_dec<kProducerRegs>();                   // the whole warpgroup (warps 9-11 are idle)
        if (warp == kConsumers / 32 && elect_one()) {
            Ring r(stages);
            if ((P.b_resident || P.res_mma) && (int)blockIdx.x < P.num_tiles) {
                // gridDim.x is a multiple of n_tiles_n, so every tile of this CTA has the same N tile
                const int nt0 = blockIdx.x % P.n_tiles_n;
                mbar_expect_tx(&bres_bar, (uint32_t)((P.b_resident ? kblocks_all * kBBytes : 0) + (P.res_mma ? 8192 : 0)));   // kblocks_all counts weight blocks
                if (P.res_mma) tma_load_2d(ident, &P.tmI, &bres_bar, 0, 0);
                if (P.b_resident)
                    for (int kb = 0; kb < kblocks_all; ++kb)
                        tma_load_2d(bres + (size_t)kb * kBBytes, &P.tmB, &bres_bar, kb * kBK, nt0 * BN);
            }
            for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
                int pi, wb, hb, ib, nt;
                decode_tile(P, tile, pi, wb, hb, ib, nt);
                const Problem &pr = P.prob[pi];
                const int w0 = wb * pr.BW * P.stride - P.pad, h0 = hb * pr.BH * P.stride - P.pad, i0 = ib * pr.BI;
                const int tap_lo = ksplit_of(P, tile) * taps_per;
                KIter it(tap_lo + taps_per, P.cin_blocks, kKMode, tap_lo);
                for (int j = 0; j < kblocks; ++j, it.next()) {
                    const int kh = it.tap / P.KW, kw = it.tap - kh * P.KW;
                    mbar_wait(&empty[r.stage], r.phase ^ 1);
                    uint8_t *sa = smem + (size_t)r.stage * kStageBytes;
                    const int wblk = ((it.tap * P.cin_blocks + it.cb) * kWTerms) * kBK;      // K offset of the (hi, lo) weight blocks
                    if constexpr (WALK == kWalkNcat) {
                        // one stage = x_hi tile | x_lo tile | w_hi block | w_lo block of this (tap, channel block)
                        mbar_expect_tx(&full[r.stage], 2 * kABytes + (P.b_resident ? 0 : 2 * kBBytes));
                        tma_load_5d(sa, &P.tmA[pi], &full[r.stage], it.cb * kBK, 0, w0 + kw, h0 + kh, i0);
                        tma_load_5d(sa + kABytes, &P.tmA[pi], &full[r.stage], it.cb * kBK, 1, w0 + kw, h0 + kh, i0);
                        if (!P.b_resident) {
                            tma_load_2d(sa + 2 * kABytes, &P.tmB, &full[r.stage], wblk, nt * BN);
                            tma_load_2d(sa + 2 * kABytes + kBBytes, &P.tmB, &full[r.stage], wblk + kBK, nt * BN);
                        }
                    } else {
                        mbar_expect_tx(&full[r.stage], P.b_resident ? kABytes : kABytes + kBBytes);
                        tma_load_5d(sa, &P.tmA[pi], &full[r.stage], it.cb * kBK, it.term == 1 ? 1 : 0, w0 + kw, h0 + kh, i0);
                        if (!P.b_resident)
                            tma_load_2d(sa + kABytes, &P.tmB, &full[r.stage], wblk + (it.term == 2 ? kBK : 0), nt * BN);
                    }
                    r.next();
                }
                if constexpr (WALK == kWalkKRes) {
                    // residual: one extra K block per 64 output channels (two in split mode: hi and lo), the A operand
                    // is the residual tile itself
                    for (int g = 0; g < BN / 64 && nt * BN + g * 64 < P.Cout; ++g)
                        for (int t = 0; t < kWTerms; ++t) {
                            mbar_wait(&empty[r.stage], r.phase ^ 1);
                            mbar_expect_tx(&full[r.stage], kABytes);
                            tma_load_5d(smem + (size_t)r.stage * kStageBytes, &P.tmRes[pi], &full[r.stage], nt * BN + g * 64, t,
                                        wb * pr.BW, hb * pr.BH, ib * pr.BI);
                            r.next();
                        }
                }
            }
        }
    } else if (DEFORM) {
        // ===================================================== deformable A-operand producers (warps 8-15)
        // Per tap: threads 0-127 compute the bilinear parameters of their output pixel (4 weights + 4 element
        // offsets, deform_conv_cuda_kernel.cu:84-115 + the validity test of :229) into a shared table; then all
        // 256 threads gather: 8 consecutive lanes fetch the 8 x 16 B of one pixel's 64-channel block for each of
        // the 4 corners (every load instruction covers whole 128-byte lines), blend in fp32, round to bf16 and
        // store to the stage in the 128-byte-swizzled K-major layout the MMA expects.
        __shared__ float4 s_w[2][128];
        __shared__ uint2 s_wh[2][128];                     // the same four weights as fp16 (split mode: blend of the lo halves)
        __shared__ int4 s_o[2][128];
        if constexpr (kFragEpi) setmaxnreg_dec<kWideProducerRegs>();
        const int pt = threadIdx.x - kConsumers;           // 0..kDP-1
        // the B tile(s) of a stage: thread 0 of the producers adds their bytes to the stage's barrier and issues the TMA loads
        auto load_b = [&](int stage, int tap, int cb, int nt) {
            uint8_t *sb = smem + (size_t)stage * kStageBytes + (P.dcat ? 2 * kABytes : kABytes);
            const int wblk = (tap * P.cin_blocks + cb) * (P.split ? 2 : 1) * kBK;
            mbar_expect_tx(&full[stage], P.dcat ? 2 * kBBytes : kBBytes);
            tma_load_2d(sb, &P.tmB, &full[stage], wblk, nt * BN);
            if (P.dcat) tma_load_2d(sb + kBBytes, &P.tmB, &full[stage], wblk + kBK, nt * BN);
        };
        Ring r(stages);
        int tb = 0;
        for (int tile = blockIdx.x; tile < P.num_tiles; tile += gridDim.x) {
            int pi, wb, hb, ib, nt;
            decode_tile(P, tile, pi, wb, hb, ib, nt);
            const Problem &pr = P.prob[pi];
            const int taps = P.KH * P.KW;
            for (int tap = 0; tap < taps; ++tap) {
                if (pt < 128) {
                    // this thread's output pixel, derived again for every tap: nothing of it stays live through the gather
                    const int iw = pt & (pr.BW - 1), ih = (pt >> pr.lbw) & (pr.BH - 1), ii = pt >> (pr.lbw + pr.lbh);
                    const int w = wb * pr.BW + iw, h = hb * pr.BH + ih, n = ib * pr.BI + ii;
                    const bool valid = (w < pr.Wo) && (h < pr.Ho) && (n < pr.N);
                    const size_t opix = ((size_t)(valid ? n : 0) * pr.Ho + (valid ? h : 0)) * pr.Wo + (valid ? w : 0);
                    const float *offp = pr.offset + opix * (2 * taps);
                    const float *mskp = pr.mask ? pr.mask + opix * taps : nullptr;
                    const int cpp = P.Cin * (SPLIT ? 2 : 1);            // 16-bit elements per pixel (hi and lo halves in split mode)
                    const int img0 = (valid ? n : 0) * pr.H * pr.W * cpp;
                    const int kh = tap / P.KW, kw = tap - kh * P.KW;
                    float4 wv = make_float4(0.f, 0.f, 0.f, 0.f);
                    int4 ov = make_int4(img0, img0, img0, img0);
                    if (valid) {
                        const float h_im = (float)(h * P.stride - P.pad + kh) + offp[2 * tap];
                        const float w_im = (float)(w * P.stride - P.pad + kw) + offp[2 * tap + 1];
                        if (h_im > -1.f && w_im > -1.f && h_im < (float)pr.H && w_im < (float)pr.W) {
                            const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
                            const int h_high = h_low + 1, w_high = w_low + 1;
                            const float lh = h_im - (float)h_low, lw = w_im - (float)w_low, hh = 1.f - lh, hw = 1.f - lw;
                            if (h_low >= 0 && w_low >= 0) { wv.x = hh * hw; ov.x = img0 + (h_low * pr.W + w_low) * cpp; }
                            if (h_low >= 0 && w_high <= pr.W - 1) { wv.y = hh * lw; ov.y = img0 + (h_low * pr.W + w_high) * cpp; }
                            if (h_high <= pr.H - 1 && w_low >= 0) { wv.z = lh * hw; ov.z = img0 + (h_high * pr.W + w_low) * cpp; }
                            if (h_high <= pr.H - 1 && w_high <= pr.W - 1) { wv.w = lh * lw; ov.w = img0 + (h_high * pr.W + w_high) * cpp; }
                            if (mskp) {
                                // DCNv2 (modulated_deformable_im2col_gpu_kernel, deform_conv_cuda_kernel.cu:570-633): the sample
                                // is multiplied by the mask value of (pixel, tap); folded into the four corner weights
                                const float m = mskp[tap];
                                wv.x *= m; wv.y *= m; wv.z *= m; wv.w *= m;
                            }
                        }
                    }
                    s_w[tb][pt] = wv;
                    s_o[tb][pt] = ov;
                    if (P.split) {
                        const __half2 w01 = __floats2half2_rn(wv.x, wv.y), w23 = __floats2half2_rn(wv.z, wv.w);
                        s_wh[tb][pt] = make_uint2(*reinterpret_cast<const uint32_t *>(&w01), *reinterpret_cast<const uint32_t *>(&w23));
                    }
                }
                asm volatile("bar.sync 2, %0;" ::"n"(kDP) : "memory");
                for (int cb = 0; cb < P.cin_blocks; ++cb) {
                    if constexpr (!SPLIT) {
                        mbar_wait(&empty[r.stage], r.phase ^ 1);
                        if (pt == 0) load_b(r.stage, tap, cb, nt);
                        uint8_t *sa = smem + (size_t)r.stage * kStageBytes;
                        uint4 u[kDItems][4];
#pragma unroll
                        for (int it = 0; it < kDItems; ++it) {
                            const int item = pt + it * kDP, row = item >> 3, c16 = item & 7;
                            const int4 ov = s_o[tb][row];
                            const int co = cb * kBK + c16 * 8;
                            u[it][0] = *reinterpret_cast<const uint4 *>(pr.x + ov.x + co);
                            u[it][1] = *reinterpret_cast<const uint4 *>(pr.x + ov.y + co);
                            u[it][2] = *reinterpret_cast<const uint4 *>(pr.x + ov.z + co);
                            u[it][3] = *reinterpret_cast<const uint4 *>(pr.x + ov.w + co);
                        }
#pragma unroll
                        for (int it = 0; it < kDItems; ++it) {
                            const int item = pt + it * kDP, row = item >> 3, c16 = item & 7;
                            const float4 wv = s_w[tb][row];
                            const uint32_t *a1 = reinterpret_cast<const uint32_t *>(&u[it][0]);
                            const uint32_t *a2 = reinterpret_cast<const uint32_t *>(&u[it][1]);
                            const uint32_t *a3 = reinterpret_cast<const uint32_t *>(&u[it][2]);
                            const uint32_t *a4 = reinterpret_cast<const uint32_t *>(&u[it][3]);
                            uint32_t pk[4];
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                const float2 f1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&a1[k]));
                                const float2 f2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&a2[k]));
                                const float2 f3 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&a3[k]));
                                const float2 f4 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&a4[k]));
                                const float vx = wv.x * f1.x + wv.y * f2.x + wv.z * f3.x + wv.w * f4.x;
                                const float vy = wv.x * f1.y + wv.y * f2.y + wv.z * f3.y + wv.w * f4.y;
                                __nv_bfloat162 b2 = __floats2bfloat162_rn(vx, vy);
                                pk[k] = *reinterpret_cast<uint32_t *>(&b2);
                            }
                            *reinterpret_cast<uint4 *>(sa + (size_t)row * 128 + ((c16 ^ (row & 7)) << 4)) = make_uint4(pk[0], pk[1], pk[2], pk[3]);
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic -> async proxy (wgmma reads smem)
                        __syncwarp();                                                   // every lane has fenced its own stores
                        if ((pt & 31) == 0) mbar_arrive(&full[r.stage]);
                        r.next();
                    } else {
                        // split mode: every corner is read as its (hi, lo) fp16 pair, the sample is formed in fp32 exactly as
                        // the reference does (deform_conv_cuda_kernel.cu:84-115), split again, and written as the x_hi and
                        // x_lo tiles of this K block's stage
                        const __half *xh = reinterpret_cast<const __half *>(pr.x);
                        auto load_item = [&](int it, uint4 (&u)[4][2]) {       // item `it` of this thread: its four corners
                            const int item = pt + it * kDP, row = item >> 3, c16 = item & 7;
                            const int4 ov = s_o[tb][row];
                            const int co = cb * kBK + c16 * 8;
                            const int oo[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
                            for (int c = 0; c < 4; ++c) {
                                u[c][0] = *reinterpret_cast<const uint4 *>(xh + oo[c] + co);
                                u[c][1] = *reinterpret_cast<const uint4 *>(xh + oo[c] + P.Cin + co);
                            }
                        };
                        auto item_at = [&](int it) {                           // its byte offset in the x_hi / x_lo tile
                            const int item = pt + it * kDP, row = item >> 3, c16 = item & 7;
                            return (uint32_t)(row * 128 + ((c16 ^ (row & 7)) << 4));
                        };
                        if constexpr (!kFragEpi) {
                            // the samples of all four items are held until the stage is free
                            uint32_t phi[kDItems][4], plo[kDItems][4];
#pragma unroll
                            for (int i2 = 0; i2 < kDItems / kDRound; ++i2) {
                                uint4 u[kDRound][4][2];
#pragma unroll
                                for (int i1 = 0; i1 < kDRound; ++i1) load_item(i2 * kDRound + i1, u[i1]);
#pragma unroll
                                for (int i1 = 0; i1 < kDRound; ++i1) {
                                    const int it = i2 * kDRound + i1, row = (pt + it * kDP) >> 3;
                                    split_sample(u[i1], s_w[tb][row], s_wh[tb][row], phi[it], plo[it]);
                                }
                            }
                            mbar_wait(&empty[r.stage], r.phase ^ 1);
                            if (pt == 0) load_b(r.stage, tap, cb, nt);
                            uint8_t *sa = smem + (size_t)r.stage * kStageBytes;
#pragma unroll
                            for (int it = 0; it < kDItems; ++it) {
                                const uint32_t at = item_at(it);
                                *reinterpret_cast<uint4 *>(sa + at) = make_uint4(phi[it][0], phi[it][1], phi[it][2], phi[it][3]);
                                *reinterpret_cast<uint4 *>(sa + kABytes + at) = make_uint4(plo[it][0], plo[it][1], plo[it][2], plo[it][3]);
                            }
                        } else {
                            // wide variant (96 registers: no room to hold the samples): the first round's loads are in
                            // flight while the stage is awaited, and every sample goes to the stage as soon as it is formed
                            const uint32_t sa = smem_u32(smem + (size_t)r.stage * kStageBytes);
#pragma unroll
                            for (int i2 = 0; i2 < kDItems / kDRound; ++i2) {
                                uint4 u[kDRound][4][2];
#pragma unroll
                                for (int i1 = 0; i1 < kDRound; ++i1) load_item(i2 * kDRound + i1, u[i1]);
                                if (i2 == 0) {
                                    mbar_wait(&empty[r.stage], r.phase ^ 1);
                                    if (pt == 0) load_b(r.stage, tap, cb, nt);
                                }
#pragma unroll
                                for (int i1 = 0; i1 < kDRound; ++i1) {
                                    const int it = i2 * kDRound + i1, row = (pt + it * kDP) >> 3;
                                    uint32_t hi[4], lo[4];
                                    split_sample(u[i1], s_w[tb][row], s_wh[tb][row], hi, lo);
                                    const uint32_t at = sa + item_at(it);
                                    sts128(at, make_uint4(hi[0], hi[1], hi[2], hi[3]));
                                    sts128(at + kABytes, make_uint4(lo[0], lo[1], lo[2], lo[3]));
                                }
                            }
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        __syncwarp();
                        if ((pt & 31) == 0) mbar_arrive(&full[r.stage]);
                        r.next();
                    }
                }
                tb ^= 1;
            }
        }
    }
}

// ----------------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult st;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &st) == cudaSuccess && st == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int pow2_floor(int v) { int p = 1; while (p * 2 <= v) p *= 2; return p; }

// event pool for orp_set_timing(1): every conv_tc launch is bracketed on its own stream
constexpr int kEvPool = 1024;
thread_local cudaEvent_t g_tc_ev[kEvPool][2];
thread_local int g_tc_ev_created = 0, g_tc_ev_used = 0;
thread_local double g_tc_flops = 0.0;
// plan of this thread's most recent launch (orp_tc_last_plan)
thread_local orp_tc_plan g_tc_plan;
thread_local bool g_tc_plan_set = false;

// shared memory one thread block of an H100 can opt into, and the static shared memory the budget sets aside for each variant
// (barriers and bias slice; the deformable producers' sample tables too).  launch_tc checks the compiled size against the plan.
constexpr int kSmemPerBlock = 227 * 1024;
constexpr int kStaticSmemPlain = 4096;
constexpr int kStaticSmemDeform = 14336;

// what a launch asks for
struct ConvDesc {
    int nprob;
    const orp_tc_problem *probs;
    const void *w;
    int Cout, Cout_padded, KH, KW, Cin, stride, pad;
    const float *bias;
    int relu, out_f32, deform;
    int split;                                // f16x3 operands (0 / 1)
    int wscale_log2;                          // f16x3: power-of-two weight scale
    int stem;                                 // 0, or 2 for conv1 in space-to-depth form (the value orp_tc_plan.stem reports)
    int ksplit;                               // split-K factor, >= 1
};

// how it runs: the plan orp_tc_last_plan reports, plus the tile geometry of every problem (Problem without its pointers)
struct ConvPlan {
    orp_tc_plan rep;
    Problem prob[kMaxProb];
    int num_m_tiles;
    int kbn;                                  // the kernel's accumulator width: BN, or 2 BN when a CTA computes an N-tile pair
    int extra_bytes;                          // dynamic shared memory beside the stages: identity, resident slab, output staging
};

// the checks that need no device (see orp_conv2d_bf16 / orp_conv2d_f16x3 in include/orp_b200.h)
int check_conv(const ConvDesc &d)
{
    if (d.split && (d.wscale_log2 < 0 || d.wscale_log2 > 15)) return fail(ORP_EINVAL, "conv2d_f16x3: weight scale exponent must be in 0..15");
    if (d.nprob < 1 || d.nprob > kMaxProb || !d.probs || !d.w) return fail(ORP_EINVAL, "conv2d_tc: bad arguments");
    if (d.Cin % 8) return fail(ORP_EINVAL, "conv2d_tc: Cin must be a multiple of 8 (16-byte channel rows)");
    if (d.deform && (d.Cin % kBK)) return fail(ORP_EINVAL, "conv2d_tc: deformable conv needs Cin % 64 == 0");
    if (d.Cout_padded % 32 || d.Cout_padded < d.Cout) return fail(ORP_EINVAL, "conv2d_tc: padded Cout must be a multiple of 32");
    // a tile spans BW * stride <= 256 input columns (the TMA box limit) with BW >= 1
    if (d.stride < 1 || d.stride > 256) return fail(ORP_EINVAL, "conv2d_tc: stride must be in 1..256");
    // the deformable producers address the input with 32-bit element offsets (img0, s_o): N*H*W*Cin*planes must stay below 2^31
    if (d.deform)
        for (int i = 0; i < d.nprob; ++i)
            if ((long long)d.probs[i].N * d.probs[i].H * d.probs[i].W * d.Cin * (d.split ? 2 : 1) >= (1LL << 31))
                return fail(ORP_EINVAL, "conv2d_tc: deformable input has 2^31 or more 16-bit elements (32-bit sample offsets)");
    const orp_tc_problem &q0 = d.probs[0];
    if (d.ksplit > 1 && (d.nprob != 1 || d.deform || d.stem || !d.out_f32 || (d.KH * d.KW) % d.ksplit || q0.residual_bf16 ||
                         q0.residual_f32 || d.bias || d.relu))
        return fail(ORP_EINVAL, "conv2d_tc: split-K serves one plain problem with an fp32 partial-sum output and taps % ksplit == 0");
    return ORP_OK;
}

// The launch plan of a convolution on a device with `sms` SMs.  Pure: no CUDA call, no environment, no global state; the
// problem pointers are only tested for NULL.
int plan_conv(const ConvDesc &d, int sms, ConvPlan &pl)
{
    int rc = check_conv(d);
    if (rc) return rc;
    memset(&pl, 0, sizeof(pl));
    const int nprob = d.nprob, ksplit = d.ksplit, T = d.split ? 2 : 1;   // T: 16-bit planes per value (hi, lo)
    const orp_tc_problem *probs = d.probs;

    int BN = 256;
    if (d.Cout_padded % 256) BN = (d.Cout_padded % 128 == 0) ? 128 : (d.Cout_padded % 64 == 0) ? 64 : 32;
    {
        // narrower accumulators when the 128 x BN tiling would leave SMs idle
        long long mtiles = 0;
        for (int i = 0; i < nprob; ++i) {
            const int ho = (probs[i].H + 2 * d.pad - (d.KH - 1) - 1) / d.stride + 1, wo = (probs[i].W + 2 * d.pad - (d.KW - 1) - 1) / d.stride + 1;
            mtiles += ((long long)probs[i].N * ho * wo + 127) / 128;
        }
        while (BN > 64 && mtiles * (d.Cout_padded / BN) * ksplit < 120) BN /= 2;
    }
    // the deformable variant's 512 threads leave 128 registers each: a 64 x 128 fp32 accumulator fragment (64 per thread)
    // fits beside the staged epilogue, a 64 x 256 one does not
    if (d.deform && BN > 128) BN = 128;
    // a partial last channel block is zero-filled by TMA (A operand) and by the weight layout (B operand)
    const int cin_blocks = (d.Cin + kBK - 1) / kBK;
    const int n_tiles_n = d.Cout_padded / BN;
    // N-tile pairs: in f16x3 with 16-bit outputs and no GELU (the detector's head) a deformable launch computes two adjacent
    // 128-wide N tiles of an M tile in one CTA, on ONE sampled A operand - every sample is gathered once per M tile instead
    // of once per N tile, half the gathered bytes.  The kernel runs them as one 256-wide tile, in the variant whose consumers
    // take registers from the producers and finish from the fragments (frag_epilogue).
    const int n_pair = (d.deform && d.split && !d.out_f32 && d.Cout % 8 == 0 && d.relu != 2 && BN == 128 && n_tiles_n % 2 == 0) ? 2 : 1;
    const int kbn = BN * n_pair;
    int mt = 0;
    for (int i = 0; i < nprob; ++i) {
        const orp_tc_problem &q = probs[i];
        Problem &pr = pl.prob[i];
        pr.N = q.N; pr.H = q.H; pr.W = q.W;
        pr.Ho = (q.H + 2 * d.pad - (d.KH - 1) - 1) / d.stride + 1;
        pr.Wo = (q.W + 2 * d.pad - (d.KW - 1) - 1) / d.stride + 1;
        if (pr.Ho <= 0 || pr.Wo <= 0 || !q.x || !q.out) return fail(ORP_EINVAL, "conv2d_tc: bad problem");
        pr.BW = pow2_floor(pr.Wo < 128 ? pr.Wo : 128);
        // the TMA box spans BW * stride columns (<= 256); BW stays a power of two, as the row decode (& (BW - 1), lbw) needs
        if (d.stride * pr.BW > 256) pr.BW = pow2_floor(256 / d.stride);
        // (measured: 16 x 8 pixel tiles for the deformable variant change nothing - 1361 vs 1334 us per f16x3 launch, and neither
        // does the spread of the offsets: the gather runs at the ~47 GB/s per SM L2 -> SM ceiling whatever its locality)
        pr.BH = pow2_floor(pr.Ho < 128 / pr.BW ? pr.Ho : 128 / pr.BW);
        pr.BI = 128 / (pr.BW * pr.BH);
        pr.lbw = 0; while ((1 << pr.lbw) < pr.BW) ++pr.lbw;
        pr.lbh = 0; while ((1 << pr.lbh) < pr.BH) ++pr.lbh;
        pr.tiles_w = ceil_div(pr.Wo, pr.BW); pr.tiles_h = ceil_div(pr.Ho, pr.BH); pr.tiles_i = ceil_div(pr.N, pr.BI);
        pr.tile_start = mt;
        pr.fd_tw.set((uint32_t)pr.tiles_w); pr.fd_th.set((uint32_t)pr.tiles_h);
        mt += pr.tiles_w * pr.tiles_h * pr.tiles_i;
        if (d.deform && !q.offset) return fail(ORP_EINVAL, "conv2d_tc: deformable conv needs offsets");
    }
    const int num_tiles = mt * n_tiles_n * ksplit;
    // TMA epilogue: 16-bit outputs whose channel count is a multiple of 64
    bool any_res = false;
    for (int i = 0; i < nprob; ++i) any_res = any_res || (probs[i].residual_bf16 != nullptr);
    // (f16x3 also takes channel counts that are only a multiple of 8 - Swin's 96 / 288: the TMA unit clips the last box)
    const int tma_epi = (!d.out_f32 && ((d.Cout % 64 == 0) || (d.split && d.Cout % 8 == 0)) && BN >= 64) ? 1 : 0;
    if (d.split && !d.out_f32 && !tma_epi) return fail(ORP_EINVAL, "conv2d_f16x3: 16-bit outputs need Cout % 8 == 0 and weights padded to a multiple of 64 rows");
    if (d.split && d.out_f32 && any_res) return fail(ORP_EINVAL, "conv2d_f16x3: fp32 outputs take an fp32 residual only");
    // GroupNorm statistics: fused into the TMA epilogue when every warp's 32 rows lie in one image
    const bool frag_epi = frag_epilogue(kbn, d.deform != 0);     // (fuses no GroupNorm statistics, merges no hi / lo tiles)
    bool want_gn = false, gn_ok = tma_epi && d.Cout == 256 && !d.bias && !d.relu && !frag_epi;
    for (int i = 0; i < nprob; ++i) {
        want_gn = want_gn || (probs[i].gn_stats != nullptr);
        if (pl.prob[i].BW * pl.prob[i].BH < 32) gn_ok = false;
    }
    const int gn_fused = (want_gn && gn_ok) ? 1 : 0;
    const bool mem_bound = any_res || (d.KH * d.KW * (d.Cin / kBK) <= 8);
    int epi_bufs = mem_bound ? 2 : 1;          // a second staging tile costs compute-bound layers a main-loop stage
    const int epi_merge = (d.split && tma_epi && !frag_epi && (mem_bound || d.stem == 2)) ? 1 : 0;
    // terms concatenated along N for narrow layers (kernel header); the residual / deformable / fp32-output variants keep
    // the K-concatenated walk
    const int dcat = (d.split && d.deform) ? 1 : 0;
    const int ncat = (d.split && tma_epi && BN <= 128 && !d.deform && !any_res) ? 1 : 0;
    // residual through the tensor core (TMA epilogue only; the staged epilogue adds it itself)
    const int res_mma = (tma_epi && any_res) ? 1 : 0;
    if (res_mma) {
        if (d.deform) return fail(ORP_EINVAL, "conv2d_tc: residual is not supported on the deformable path");
        for (int i = 0; i < nprob; ++i)
            if (!probs[i].residual_bf16) return fail(ORP_EINVAL, "conv2d_tc: residual must be given for every problem or none");
    }
    // layers whose whole weight slab for one N tile is <= 72 KiB keep it resident; stages then carry only the A tile
    const int slab_bytes = d.KH * d.KW * T * cin_blocks * BN * kBK * 2;
    int b_resident = (!d.deform && ksplit == 1 && slab_bytes <= 72 * 1024) ? 1 : 0;
    int grid = num_tiles / n_pair < sms ? num_tiles / n_pair : sms;      // a CTA takes an N-tile pair at a time
    if (b_resident && grid >= n_tiles_n) grid -= grid % n_tiles_n;       // fixed N tile per CTA
    else if (b_resident) b_resident = 0;
    // shared-memory budget: staged accumulator pass + output staging + resident weights + main-loop stages.  When the extras
    // leave fewer than three stages they are given up in order of least value: the second staging slot, the resident slab.
    int stage_b = 0, extra = 0, stages = 0;
    for (;;) {
        stage_b = stage_bytes(kbn, ncat || dcat, b_resident);
        const int hc = BN < 64 ? BN : 64;
        int staging = d.out_f32 ? 0 : 128 * (hc * 2 + 16);
        if (tma_epi) staging = epi_bufs * (epi_merge ? 32768 : 16384);
        extra = (res_mma ? 8192 : 0) + (b_resident ? slab_bytes : 0) + staging;
        stages = (kSmemPerBlock - (d.deform ? kStaticSmemDeform : kStaticSmemPlain) - dyn_smem_bytes(stage_b, 0, extra, frag_epi)) / stage_b;
        if (stages >= 3) break;
        if (epi_bufs == 2) { epi_bufs = 1; continue; }
        if (b_resident) { b_resident = 0; continue; }
        if (stages >= 2) break;
        return fail(ORP_EINVAL, "conv2d_tc: shared-memory budget cannot hold two main-loop stages");
    }
    if (stages > kStagesMax) stages = kStagesMax;
    if (d.deform && stages > 3) stages = 3;     // leave L1 capacity for the bilinear gather (corner reuse between neighbouring pixels)

    pl.num_m_tiles = mt;
    pl.kbn = kbn;
    pl.extra_bytes = extra;
    orp_tc_plan &r = pl.rep;
    r.BN = BN; r.stages = stages; r.grid = grid; r.num_tiles = num_tiles; r.n_tiles_n = n_tiles_n;
    r.ksplit = ksplit; r.nprob = nprob; r.Cout = d.Cout; r.Cout_padded = d.Cout_padded;
    r.split = d.split ? 1 : 0; r.deform = d.deform ? 1 : 0; r.out_f32 = d.out_f32 ? 1 : 0; r.stem = d.stem; r.relu = d.relu;
    r.bias = d.bias ? 1 : 0;
    for (int i = 0; i < nprob; ++i) {
        if (probs[i].residual_bf16) r.residual = 1;
        else if (probs[i].residual_f32) r.residual = 2;
        r.BW[i] = pl.prob[i].BW; r.BH[i] = pl.prob[i].BH; r.BI[i] = pl.prob[i].BI;
    }
    r.tma_epi = tma_epi; r.ncat = ncat; r.dcat = dcat; r.res_mma = res_mma; r.b_resident = b_resident;
    r.epi_merge = epi_merge; r.epi_bufs = epi_bufs; r.gn_fused = gn_fused; r.n_pair = n_pair;
    return ORP_OK;
}

// the kernel's parameter block of a plan, tensor maps aside
int make_params(const ConvDesc &d, const ConvPlan &pl, TcParams &P)
{
    memset(&P, 0, sizeof(P));
    P.nprob = d.nprob; P.KH = d.KH; P.KW = d.KW; P.Cin = d.Cin; P.cin_blocks = (d.Cin + kBK - 1) / kBK;
    P.stride = d.stride; P.pad = d.pad;
    P.Cout = d.Cout; P.relu = d.relu; P.bias = d.bias; P.s2d_stem = (d.stem == 2) ? 1 : 0;
    P.split = d.split ? 1 : 0;
    P.oscale = d.split ? ldexpf(1.f, -d.wscale_log2) : 1.f;
    {
        void *ovf = nullptr;
        ORP_CUDA(cudaGetSymbolAddress(&ovf, g_f16_overflow));
        P.ovf = static_cast<unsigned int *>(ovf);
    }
    P.n_tiles_n = pl.rep.n_tiles_n / pl.rep.n_pair;              // the kernel's N tiles are kbn wide
    P.fd_ntn.set((uint32_t)P.n_tiles_n);
    for (int i = 0; i < d.nprob; ++i) {
        const orp_tc_problem &q = d.probs[i];
        Problem &pr = P.prob[i];
        pr = pl.prob[i];
        pr.out = q.out; pr.res = static_cast<const __nv_bfloat16 *>(q.residual_bf16); pr.res32 = q.residual_f32;
        pr.x = static_cast<const __nv_bfloat16 *>(q.x); pr.offset = q.offset; pr.gn_stats = q.gn_stats; pr.mask = q.mask;
    }
    P.num_m_tiles = pl.num_m_tiles;
    P.num_tiles = pl.rep.num_tiles / pl.rep.n_pair;
    P.ksplit = d.ksplit;
    P.fd_ks.set((uint32_t)d.ksplit);
    P.ks_stride = (long long)P.prob[0].N * P.prob[0].Ho * P.prob[0].Wo * d.Cout;
    P.tma_epi = pl.rep.tma_epi; P.epi_bufs = pl.rep.epi_bufs; P.epi_merge = pl.rep.epi_merge; P.ncat = pl.rep.ncat;
    P.b_resident = pl.rep.b_resident; P.res_mma = pl.rep.res_mma; P.gn_fused = pl.rep.gn_fused; P.dcat = pl.rep.dcat;
    return ORP_OK;
}

// the tensor maps of a launch: A (plain variant), B, the identity (res_mma), output and residual (TMA epilogue)
int encode_maps(const ConvDesc &d, const ConvPlan &pl, TcParams &P)
{
    EncodeTiledFn enc = encode_fn();
    if (!enc) return fail(ORP_ECUDA, "conv2d_tc: cuTensorMapEncodeTiled unavailable");
    const CUtensorMapDataType dt16 = d.split ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    const int T = d.split ? 2 : 1, Cin = d.Cin, Cout = d.Cout, stride = d.stride;
    if (!d.deform) {
        for (int i = 0; i < d.nprob; ++i) {
            const orp_tc_problem &q = d.probs[i];
            const Problem &pr = P.prob[i];
            // 5-D view {channel, plane (hi / lo), w, h, image}; bf16 tensors have a single plane.  Split activations are
            // [N,H,W,2,C]: the lo plane of a pixel follows its hi plane.
            cuuint64_t gdim[5] = {(cuuint64_t)Cin, (cuuint64_t)T, (cuuint64_t)q.W, (cuuint64_t)q.H, (cuuint64_t)q.N};
            cuuint64_t gstr[4] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cin * 2 * T, (cuuint64_t)q.W * Cin * 2 * T,
                                  (cuuint64_t)q.H * q.W * Cin * 2 * T};
            if (d.stem == 2) {
                // space-to-depth stem: the tensor is [T][N, H, W + 3, 16] (planes outermost); a 64-element "pixel" row of
                // the GEMM is the 4 horizontally adjacent 16-channel pixels starting at w, so consecutive w overlap
                // (stride 32 bytes)
                gstr[0] = (cuuint64_t)q.N * q.H * (q.W + 3) * 32;
                gstr[1] = 32;
                gstr[2] = (cuuint64_t)(q.W + 3) * 32;
                gstr[3] = (cuuint64_t)q.H * (q.W + 3) * 32;
            }
            cuuint32_t box[5] = {(cuuint32_t)kBK, 1u, (cuuint32_t)(pr.BW * stride), (cuuint32_t)(pr.BH * stride), (cuuint32_t)pr.BI};
            cuuint32_t estr[5] = {1, 1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
            CUresult r = enc(&P.tmA[i], dt16, 5, const_cast<void *>(q.x), gdim, gstr, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return fail(ORP_ECUDA, "conv2d_tc: cuTensorMapEncodeTiled(A) failed");
        }
    }
    {
        // weights [Cout_padded][tap][cin_blocks][T][64] (zero padded per tap; T = 2: the hi block, then the lo block)
        const cuuint64_t K = (cuuint64_t)d.KH * d.KW * T * P.cin_blocks * kBK;
        cuuint64_t gdim[2] = {K, (cuuint64_t)d.Cout_padded};
        cuuint64_t gstr[1] = {K * 2};
        cuuint32_t box[2] = {(cuuint32_t)kBK, (cuuint32_t)pl.kbn};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&P.tmB, dt16, 2, const_cast<void *>(d.w), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(ORP_ECUDA, "conv2d_tc: cuTensorMapEncodeTiled(B) failed");
    }
    if (P.res_mma) {
        void *ident_ptr = nullptr;
        if (d.split) {
            ORP_CUDA(cudaGetSymbolAddress(&ident_ptr, g_ident16));
            ident_ptr = static_cast<char *>(ident_ptr) + (size_t)d.wscale_log2 * 8192;
        } else {
            ORP_CUDA(cudaGetSymbolAddress(&ident_ptr, g_ident));
        }
        cuuint64_t gdim[2] = {64, 64};
        cuuint64_t gstr[1] = {128};
        cuuint32_t box[2] = {64, 64};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&P.tmI, dt16, 2, ident_ptr, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(ORP_ECUDA, "conv2d_tc: cuTensorMapEncodeTiled(identity) failed");
    }
    if (P.tma_epi) {
        for (int i = 0; i < d.nprob; ++i) {
            const Problem &pr = P.prob[i];
            cuuint64_t gdim[5] = {(cuuint64_t)Cout, (cuuint64_t)T, (cuuint64_t)pr.Wo, (cuuint64_t)pr.Ho, (cuuint64_t)pr.N};
            cuuint64_t gstr[4] = {(cuuint64_t)Cout * 2, (cuuint64_t)Cout * 2 * T, (cuuint64_t)pr.Wo * Cout * 2 * T,
                                  (cuuint64_t)pr.Ho * pr.Wo * Cout * 2 * T};
            cuuint32_t box[5] = {64u, 1u, (cuuint32_t)pr.BW, (cuuint32_t)pr.BH, (cuuint32_t)pr.BI};
            cuuint32_t estr[5] = {1, 1, 1, 1, 1};
            CUresult r = enc(&P.tmOut[i], dt16, 5, pr.out, gdim, gstr, box, estr,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) return fail(ORP_ECUDA, "conv2d_tc: cuTensorMapEncodeTiled(out) failed");
            if (pr.res) {
                r = enc(&P.tmRes[i], dt16, 5, const_cast<__nv_bfloat16 *>(pr.res), gdim, gstr, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
                if (r != CUDA_SUCCESS) return fail(ORP_ECUDA, "conv2d_tc: cuTensorMapEncodeTiled(residual) failed");
            }
        }
    }
    return ORP_OK;
}

template <int BN, bool OUT_F32, bool DEFORM, bool SPLIT, int WALK>
int launch_tc(const TcParams &P, int stages, int grid, cudaStream_t st, int extra_bytes)
{
    constexpr bool kCat = WALK == kWalkNcat || WALK == kWalkDcat;
    const int smem = dyn_smem_bytes(stage_bytes(BN, kCat, P.b_resident), stages, extra_bytes, frag_epilogue(BN, DEFORM));
    auto kern = conv_tc_kernel<BN, OUT_F32, DEFORM, SPLIT, WALK>;
    static int smem_max = -1;                  // dynamic shared memory beside this instantiation's static shared memory
    if (smem_max < 0) {
        cudaFuncAttributes fa;
        ORP_CUDA(cudaFuncGetAttributes(&fa, kern));
        ORP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemPerBlock - (int)fa.sharedSizeBytes));
        smem_max = kSmemPerBlock - (int)fa.sharedSizeBytes;
    }
    if (smem > smem_max) {
        char need[32];
        snprintf(need, sizeof(need), "%d", smem);
        return fail(ORP_EINVAL, "conv2d_tc: the plan's %s bytes of dynamic shared memory do not fit beside the static shared memory of %s",
                    need, __PRETTY_FUNCTION__);
    }
    int slot = -1;
    if (g_timing && g_tc_ev_used < kEvPool) {
        slot = g_tc_ev_used++;
        if (slot >= g_tc_ev_created) {
            ORP_CUDA(cudaEventCreate(&g_tc_ev[slot][0]));
            ORP_CUDA(cudaEventCreate(&g_tc_ev[slot][1]));
            g_tc_ev_created = slot + 1;
        }
        ORP_CUDA(cudaEventRecord(g_tc_ev[slot][0], st));
        double fl = 0;
        for (int i = 0; i < P.nprob; ++i)
            fl += 2.0 * P.prob[i].N * P.prob[i].Ho * P.prob[i].Wo * (double)P.Cout *
                  (P.s2d_stem ? 147.0 : (double)P.KH * P.KW * P.Cin);   // algorithmic K, not the padded one
        g_tc_flops += fl;
    }
    {
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3((unsigned)grid);
        cfg.blockDim = dim3(DEFORM ? (unsigned)(kConsumers + kDP) : (unsigned)(kConsumers + 128));
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        ORP_CUDA(cudaLaunchKernelEx(&cfg, kern, P, stages));
    }
    ORP_LAUNCHED();
    if (slot >= 0) ORP_CUDA(cudaEventRecord(g_tc_ev[slot][1], st));
    return ORP_OK;
}

// the instantiation that runs a plan: operand type (P.split) and main-loop walk (P.ncat, P.dcat, P.res_mma) are
// compile-time
template <int BN, bool OUT_F32, bool DEFORM>
int launch_plan(const TcParams &P, int stages, int grid, cudaStream_t st, int extra_bytes)
{
    if constexpr (DEFORM) {
        if (P.dcat != P.split || P.ncat || P.res_mma) return fail(ORP_EINVAL, "conv2d_tc: deformable plan outside dcat == split");
        if constexpr (frag_epilogue(BN, true)) {
            if (!P.split || OUT_F32 || !P.tma_epi || P.epi_merge || P.gn_fused || P.relu == 2)
                return fail(ORP_EINVAL, "conv2d_tc: deformable N-tile pair outside f16x3 with an unmerged TMA epilogue and no GELU");
            return launch_tc<BN, false, true, true, kWalkDcat>(P, stages, grid, st, extra_bytes);
        } else {
            return P.split ? launch_tc<BN, OUT_F32, true, true, kWalkDcat>(P, stages, grid, st, extra_bytes)
                           : launch_tc<BN, OUT_F32, true, false, kWalkK>(P, stages, grid, st, extra_bytes);
        }
    } else {
        if (P.ncat && P.res_mma) return fail(ORP_EINVAL, "conv2d_tc: ncat plan with a residual");
        if (P.ncat) {
            if constexpr (!OUT_F32 && BN >= 64 && BN <= 128) {
                if (P.split) return launch_tc<BN, false, false, true, kWalkNcat>(P, stages, grid, st, extra_bytes);
            }
            return fail(ORP_EINVAL, "conv2d_tc: ncat plan outside f16x3 TMA-epilogue layers with BN 64..128");
        }
        if (P.res_mma) {
            if constexpr (!OUT_F32 && BN >= 64)
                return P.split ? launch_tc<BN, false, false, true, kWalkKRes>(P, stages, grid, st, extra_bytes)
                               : launch_tc<BN, false, false, false, kWalkKRes>(P, stages, grid, st, extra_bytes);
            return fail(ORP_EINVAL, "conv2d_tc: residual K blocks outside TMA-epilogue layers with BN >= 64");
        }
        return P.split ? launch_tc<BN, OUT_F32, false, true, kWalkK>(P, stages, grid, st, extra_bytes)
                       : launch_tc<BN, OUT_F32, false, false, kWalkK>(P, stages, grid, st, extra_bytes);
    }
}

// the kernel's accumulator width as a template argument (the deformable variant is built up to 128, and 256 wide for the
// N-tile pairs of f16x3 with 16-bit outputs)
template <bool OUT_F32, bool DEFORM>
int launch_bn(const TcParams &P, const ConvPlan &pl, cudaStream_t st)
{
    const int s = pl.rep.stages, g = pl.rep.grid, e = pl.extra_bytes;
    switch (pl.kbn) {
    case 256:
        if constexpr (!DEFORM || !OUT_F32) return launch_plan<256, OUT_F32, DEFORM>(P, s, g, st, e);
        break;
    case 128: return launch_plan<128, OUT_F32, DEFORM>(P, s, g, st, e);
    case 64: return launch_plan<64, OUT_F32, DEFORM>(P, s, g, st, e);
    case 32: return launch_plan<32, OUT_F32, DEFORM>(P, s, g, st, e);
    }
    return fail(ORP_EINVAL, "conv2d_tc: unsupported tile width");
}

// One tensor-core convolution: plan, parameter block and tensor maps, the launch, then the GroupNorm statistics the epilogue
// could not fuse.
int conv2d_tc(const ConvDesc &d, void *stream)
{
    int rc = check_conv(d);                    // argument errors come before any device work
    if (rc) return rc;
    rc = ensure_device();
    if (rc) return rc;
    int sms = 0;
    rc = device_sms(sms);
    if (rc) return rc;
    ConvPlan pl;
    rc = plan_conv(d, sms, pl);
    if (rc) return rc;
    TcParams P;
    rc = make_params(d, pl, P);
    if (rc) return rc;
    rc = encode_maps(d, pl, P);
    if (rc) return rc;
    g_tc_plan = pl.rep;
    g_tc_plan_set = true;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    rc = d.out_f32 ? (d.deform ? launch_bn<true, true>(P, pl, st) : launch_bn<true, false>(P, pl, st))
                   : (d.deform ? launch_bn<false, true>(P, pl, st) : launch_bn<false, false>(P, pl, st));
    if (rc) return rc;
    bool want_gn = false;
    for (int i = 0; i < d.nprob; ++i) want_gn = want_gn || (d.probs[i].gn_stats != nullptr);
    if (want_gn && !P.gn_fused) {
        // statistics requested but not fusable for this shape: separate pass over the bf16 output
        if (d.out_f32 || d.Cout != 256) return fail(ORP_EINVAL, "conv2d_tc: gn_stats needs a 16-bit output with 256 channels");
        for (int i = 0; i < d.nprob; ++i)
            if (d.probs[i].gn_stats) {
                int r2 = d.split ? orp_gn_stats_f16x3(P.prob[i].out, P.prob[i].N, P.prob[i].Ho * P.prob[i].Wo, 256, 32, d.probs[i].gn_stats, stream)
                                 : orp_gn_stats_bf16(P.prob[i].out, P.prob[i].N, P.prob[i].Ho * P.prob[i].Wo, 256, 32, d.probs[i].gn_stats, stream);
                if (r2) return r2;
            }
    }
    return ORP_OK;
}

// conv1 in space-to-depth form over N images of H x W: 4 x 1 taps over the rows of the [N, H/2+3, W/2+3, 16] input, each row
// read as W/2 "pixels" of 64 virtual channels (4 horizontally adjacent pixels), stride 1, no padding
int stem_desc(const void *x_s2d, int N, int H, int W, const void *w, const float *bias, int relu, void *out, int split,
              int wscale_log2, orp_tc_problem &q, ConvDesc &d)
{
    if (!x_s2d || !w || !out || N < 1 || H < 2 || W < 2 || (H & 1) || (W & 1))
        return fail(ORP_EINVAL, "stem_conv_s2d_%s: needs even H, W", split ? "f16x3" : "bf16");
    if (split && (wscale_log2 < 0 || wscale_log2 > 15)) return fail(ORP_EINVAL, "stem_conv_s2d_f16x3: weight scale exponent must be in 0..15");
    memset(&q, 0, sizeof(q));
    q.x = x_s2d;
    q.N = N; q.H = H / 2 + 3; q.W = W / 2; q.out = out;
    d = ConvDesc{1, &q, w, 64, 64, 4, 1, 64, 1, 0, bias, relu, 0, 0, split, split ? wscale_log2 : 0, 2, 1};
    return ORP_OK;
}

// the launch inside orp_conv2d_tc_splitk: fp32 partial sums into the workspace, no bias, no activation, no statistics
int splitk_desc(const orp_tc_problem *prob, const void *w, int Cout, int Cout_padded, int KH, int KW, int Cin, int stride, int pad,
                int f16x3, int wscale_log2, int ksplit, void *workspace, orp_tc_problem &q, ConvDesc &d, int &Ho, int &Wo)
{
    if (!prob || !w || !workspace || ksplit < 2 || (Cout % 8)) return fail(ORP_EINVAL, "conv2d_tc_splitk: bad arguments");
    if (f16x3 && (wscale_log2 < 0 || wscale_log2 > 15)) return fail(ORP_EINVAL, "conv2d_tc_splitk: weight scale exponent must be in 0..15");
    Ho = (prob->H + 2 * pad - (KH - 1) - 1) / stride + 1;
    Wo = (prob->W + 2 * pad - (KW - 1) - 1) / stride + 1;
    if (Ho <= 0 || Wo <= 0) return fail(ORP_EINVAL, "conv2d_tc_splitk: bad problem");
    q = *prob;                                  // every (pixel, channel, split) element of the workspace is written
    q.out = workspace;
    q.gn_stats = nullptr;
    d = ConvDesc{1, &q, w, Cout, Cout_padded, KH, KW, Cin, stride, pad, nullptr, 0, 1, 0, f16x3 ? 1 : 0, wscale_log2, 0, ksplit};
    return ORP_OK;
}

// split-K finish: fp32 sums [pixels, C] -> + bias -> ReLU -> bf16 [pixels, C] or split fp16 [pixels, 2, C]
__global__ void __launch_bounds__(256)
splitk_finish_kernel(const float *__restrict__ ws, int ksplit, size_t pixels, int C, const float *__restrict__ bias, int relu, int split,
                     void *__restrict__ out, unsigned int *ovf)
{
    const int c8 = C / 8;
    const size_t total = pixels * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t pix = i / c8;
        const int c = (int)(i - pix * c8) * 8;
        float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int k = 0; k < ksplit; ++k) {                       // fixed order: the sum is reproducible bit for bit
            const float *p = ws + (size_t)k * pixels * C + pix * C + c;
            const float4 a = *reinterpret_cast<const float4 *>(p), b = *reinterpret_cast<const float4 *>(p + 4);
            v[0] += a.x; v[1] += a.y; v[2] += a.z; v[3] += a.w; v[4] += b.x; v[5] += b.y; v[6] += b.z; v[7] += b.w;
        }
        float amax = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (bias) v[j] += bias[c + j];
            if (relu) v[j] = fmaxf(v[j], 0.f);
            amax = fmaxf(amax, fabsf(v[j]));
        }
        uint32_t hi[4], lo[4];
        if (split) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const __half2 h2 = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
                const float2 hf = __half22float2(h2);
                const __half2 l2 = __floats2half2_rn(v[2 * k] - hf.x, v[2 * k + 1] - hf.y);
                hi[k] = *reinterpret_cast<const uint32_t *>(&h2);
                lo[k] = *reinterpret_cast<const uint32_t *>(&l2);
            }
            __half *o = static_cast<__half *>(out) + pix * 2 * C + c;
            *reinterpret_cast<uint4 *>(o) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<uint4 *>(o + C) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            if (amax > 65504.f) atomicAdd(ovf, 1u);
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                __nv_bfloat162 b2 = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
                hi[k] = *reinterpret_cast<uint32_t *>(&b2);
            }
            *reinterpret_cast<uint4 *>(static_cast<__nv_bfloat16 *>(out) + pix * C + c) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        }
    }
}
}  // namespace
}  // namespace orp

using namespace orp;

extern "C" int orp_tc_timing_collect(float *total_ms, int *launches, double *flops)
{
    if (!total_ms || !launches || !flops) return fail(ORP_EINVAL, "orp_tc_timing_collect: null");
    float sum = 0.f;
    for (int i = 0; i < g_tc_ev_used; ++i) {
        float ms = 0.f;
        ORP_CUDA(cudaEventSynchronize(g_tc_ev[i][1]));
        ORP_CUDA(cudaEventElapsedTime(&ms, g_tc_ev[i][0], g_tc_ev[i][1]));
        sum += ms;
    }
    *total_ms = sum; *launches = g_tc_ev_used; *flops = g_tc_flops;
    g_tc_ev_used = 0; g_tc_flops = 0.0;
    return ORP_OK;
}

/* see include/orp_b200.h */
extern "C" int orp_tc_last_plan(orp_tc_plan *out)
{
    if (!out) return fail(ORP_EINVAL, "orp_tc_last_plan: null");
    if (!g_tc_plan_set) return fail(ORP_EINVAL, "orp_tc_last_plan: no tensor-core convolution launched on this thread");
    *out = g_tc_plan;
    return ORP_OK;
}

/* see include/orp_b200.h */
extern "C" int orp_tc_plan_conv(int nprob, const orp_tc_problem *probs, const void *w, int Cout, int Cout_padded, int KH, int KW,
                                int Cin, int stride, int pad, const float *bias, int wscale_log2, int relu, int out_f32, int deform,
                                int split, int stem, int ksplit, int sms, orp_tc_plan *out)
{
    if (!out || sms < 1 || (stem != 0 && stem != 2)) return fail(ORP_EINVAL, "orp_tc_plan_conv: bad arguments");
    split = split ? 1 : 0;
    orp_tc_problem q;
    ConvDesc d;
    int rc = ORP_OK;
    if (stem == 2 || ksplit > 1) {
        // one problem: the stem's carries the image's N, H, W; split-K's output stands in for the workspace
        if (nprob != 1 || !probs || deform || out_f32 || (stem == 2 && ksplit > 1))
            return fail(ORP_EINVAL, "orp_tc_plan_conv: the stem and split-K plan one problem with a 16-bit output");
        int Ho, Wo;
        rc = stem == 2 ? stem_desc(probs->x, probs->N, probs->H, probs->W, w, bias, relu, probs->out, split, wscale_log2, q, d)
                       : splitk_desc(probs, w, Cout, Cout_padded, KH, KW, Cin, stride, pad, split, wscale_log2, ksplit, probs->out, q,
                                     d, Ho, Wo);
    } else {
        d = ConvDesc{nprob, probs, w, Cout, Cout_padded, KH, KW, Cin, stride, pad, bias, relu, out_f32, deform, split, wscale_log2, 0, 1};
    }
    if (rc) return rc;
    ConvPlan pl;
    rc = plan_conv(d, sms, pl);
    if (rc) return rc;
    *out = pl.rep;
    return ORP_OK;
}

/* see include/orp_b200.h */
extern "C" int orp_conv2d_bf16(int nprob, const orp_tc_problem *probs, const void *w, int Cout, int Cout_padded, int KH,
                               int KW, int Cin, int stride, int pad, const float *bias, int relu, int out_f32,
                               int deform, void *stream)
{
    return conv2d_tc(ConvDesc{nprob, probs, w, Cout, Cout_padded, KH, KW, Cin, stride, pad, bias, relu, out_f32, deform, 0, 0, 0, 1},
                     stream);
}

/* see include/orp_b200.h */
extern "C" int orp_conv2d_f16x3(int nprob, const orp_tc_problem *probs, const void *w_split, int Cout, int Cout_padded, int KH,
                                int KW, int Cin, int stride, int pad, const float *bias, int wscale_log2, int relu,
                                int out_f32, int deform, void *stream)
{
    return conv2d_tc(ConvDesc{nprob, probs, w_split, Cout, Cout_padded, KH, KW, Cin, stride, pad, bias, relu, out_f32, deform, 1,
                              wscale_log2, 0, 1},
                     stream);
}

extern "C" int orp_stem_conv_s2d_f16x3(const void *x_s2d, int N, int H, int W, const void *w_split, const float *bias,
                                       int wscale_log2, int relu, void *out, void *stream)
{
    orp_tc_problem q;
    ConvDesc d;
    const int rc = stem_desc(x_s2d, N, H, W, w_split, bias, relu, out, 1, wscale_log2, q, d);
    return rc ? rc : conv2d_tc(d, stream);
}

extern "C" int orp_stem_conv_s2d_bf16(const void *x_s2d, int N, int H, int W, const void *w256, const float *bias, int relu,
                                      void *out, void *stream)
{
    orp_tc_problem q;
    ConvDesc d;
    const int rc = stem_desc(x_s2d, N, H, W, w256, bias, relu, out, 0, 0, q, d);
    return rc ? rc : conv2d_tc(d, stream);
}

// one read of the overflow counter in stream order; with reset, read and zero are one atomic exchange, so saturations
// that a launch on another stream adds meanwhile stay in the counter for the next read
__global__ void overflow_take_kernel(unsigned int *dst, int reset)
{
    *dst = reset ? atomicExch(&g_f16_overflow, 0u) : atomicAdd(&g_f16_overflow, 0u);
}

/* see include/orp_b200.h */
extern "C" int orp_f16x3_overflow_count(unsigned int *count, int reset, void *stream)
{
    if (!count) return fail(ORP_EINVAL, "f16x3_overflow_count: null");
    static thread_local unsigned int *host = nullptr;              // mapped pinned word the kernel writes
    static thread_local unsigned int *dev = nullptr;
    if (!host) {
        ORP_CUDA(cudaHostAlloc(reinterpret_cast<void **>(&host), sizeof(unsigned int), cudaHostAllocMapped));
        ORP_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void **>(&dev), host, 0));
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    overflow_take_kernel<<<1, 1, 0, st>>>(dev, reset ? 1 : 0);
    ORP_LAUNCHED();
    ORP_CUDA(cudaStreamSynchronize(st));
    *count = *host;
    return ORP_OK;
}

/* see include/orp_b200.h */
extern "C" int orp_conv2d_tc_splitk(const orp_tc_problem *prob, const void *w, int Cout, int Cout_padded, int KH, int KW, int Cin,
                                    int stride, int pad, const float *bias, int f16x3, int wscale_log2, int relu, int ksplit,
                                    float *workspace, void *stream)
{
    orp_tc_problem q;
    ConvDesc d;
    int Ho = 0, Wo = 0;
    int rc = splitk_desc(prob, w, Cout, Cout_padded, KH, KW, Cin, stride, pad, f16x3, wscale_log2, ksplit, workspace, q, d, Ho, Wo);
    if (rc) return rc;
    rc = conv2d_tc(d, stream);
    if (rc) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t pixels = (size_t)prob->N * Ho * Wo;
    void *ovf = nullptr;
    ORP_CUDA(cudaGetSymbolAddress(&ovf, g_f16_overflow));
    splitk_finish_kernel<<<grid_for(pixels * (Cout / 8), 256), 256, 0, st>>>(workspace, ksplit, pixels, Cout, bias, relu, f16x3 ? 1 : 0, prob->out,
                                                                static_cast<unsigned int *>(ovf));
    ORP_LAUNCHED();
    if (prob->gn_stats) {
        if (Cout != 256) return fail(ORP_EINVAL, "conv2d_tc_splitk: gn_stats needs 256 output channels");
        return f16x3 ? orp_gn_stats_f16x3(prob->out, prob->N, Ho * Wo, 256, 32, prob->gn_stats, stream)
                     : orp_gn_stats_bf16(prob->out, prob->N, Ho * Wo, 256, 32, prob->gn_stats, stream);
    }
    return ORP_OK;
}
