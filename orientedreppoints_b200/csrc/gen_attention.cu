// gen_attention.cu - the generalized attention block of ResNet backbones (include/orp_b200_attention.h,
// mmdet/ops/generalized_attention.py with spatial_range = -1, q_stride = 1), in the three formats of the engines.
//
// One CTA per (query tile, head, image).  Key / value tiles stream through shared memory with an fp32 online softmax and
// fp32 accumulation: the [queries x keys] energy never leaves the chip.  The position term depends on the coordinate
// difference only, so a CTA first evaluates, per query q of its tile, Tx[q][kx] = Qp[q] . Px[qx - s kx] for the Wk key
// columns and Ty[q][ky] likewise (on the tensor cores: the tile's Qp times every row of the table, each product scattered
// to the one (q, kx) it serves), and then adds Tx[q][kx] + Ty[q][ky] to each key's logit by a shared-memory gather.
//
// Tensor-core forms (bf16, f16x3): four warps, each 16 query rows, mma.sync m16n8k16 as in swin.cu's window attention;
// f16x3 evaluates every product as lo*hi + hi*lo + hi*hi of the stored fp16 pairs and splits the probabilities into a pair
// in registers.  fp32 form: one thread per query on the CUDA cores, the same sums in the same order per key.
#include <math.h>

#include "hrnet.cuh"
#include "../../include/orp_b200_attention.h"

namespace orp {
namespace {

constexpr int kTile = 64;                  // queries per CTA, keys per streamed tile, table rows per position step
constexpr int kTcThreads = 128;            // four warps x 16 query rows
constexpr int kF32Threads = 64;            // one query per thread
constexpr int kMaxSmem = 227 * 1024;       // dynamic shared memory of one sm_90 CTA

__device__ __forceinline__ void cp16(void *smem, const void *g, bool valid)
{
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(g), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_wait_all()
{
    asm volatile("cp.async.commit_group;\ncp.async.wait_all;" ::: "memory");
}
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
// (x, y) -> packed 16-bit pair of the format and the packed remainder pair
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

struct GaParams {
    const void *qc, *qp, *k, *v, *px, *py;
    void *out;
    int N, H, W, Hk, Wk, s, C, heads, ldq, ldkv;
};

// shared-memory layout of both forms: operand tiles, then the per-tile key coordinates, then Tx [kTile][Wk + 1] and
// Ty [kTile][Hk + 1] (fp32; the +1 pitch spreads a fragment's 8 rows over the banks)
template <int D> struct GaShape {
    static constexpr int kPitch = D + 8;                      // 16-bit row pitch: 80 / 144 B, conflict-free ldmatrix rows
    static constexpr int tc_tiles_bytes(bool split) { return 3 * (split ? 2 : 1) * kTile * kPitch * 2; }   // Q | K | V
    static constexpr int f32_tiles_bytes() { return 2 * kTile * D * 4; }                                  // K | V
};
inline int tables_bytes(const GaParams &p) { return p.px ? kTile * ((p.Wk + 1) + (p.Hk + 1)) * 4 : 0; }

// rows [r0, r0 + kTile) of a token tensor (pitch ld, NP planes) -> dst [NP][kTile][PITCH] 16-bit; rows >= nrows are zero
template <int NP, int D>
__device__ __forceinline__ void stage_rows(uint16_t *dst, const uint16_t *src, long long r0, int nrows, int ld, int col0)
{
    constexpr int kC8 = D / 8, kPitch = GaShape<D>::kPitch;
    for (int i = threadIdx.x; i < kTile * NP * kC8; i += kTcThreads) {
        const int c8 = i % kC8, rest = i / kC8, pl = rest % NP, row = rest / NP;
        const bool valid = row < nrows;
        const uint16_t *g = valid ? src + ((r0 + row) * NP + pl) * (long long)ld + col0 + c8 * 8 : src;
        cp16(dst + (pl * kTile + row) * kPitch + c8 * 8, g, valid);
    }
}

// S[16 x 64] of this warp = A (16 rows of D, fragments a) times the kTile staged rows of sb, in the format's products
template <bool SPLIT, int D>
__device__ __forceinline__ void mma_rows(float (&sc)[8][4], const uint32_t (&a)[SPLIT ? 2 : 1][D / 16][4], const uint16_t *sb, int lane)
{
    constexpr int NP = SPLIT ? 2 : 1, kPitch = GaShape<D>::kPitch;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
#pragma unroll
        for (int h = 0; h < D / 32; ++h) {
            uint32_t b[NP][4];
#pragma unroll
            for (int pl = 0; pl < NP; ++pl) ldsm_x4(b[pl], sb + (pl * kTile + 8 * j + (lane & 7)) * kPitch + h * 32 + (lane >> 3) * 8);
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                const int ks = 2 * h + kk;
                if (SPLIT) {
                    mma16816<SPLIT>(sc[j], a[NP - 1][ks], b[0][2 * kk], b[0][2 * kk + 1]);       // lo x hi
                    mma16816<SPLIT>(sc[j], a[0][ks], b[NP - 1][2 * kk], b[NP - 1][2 * kk + 1]);  // hi x lo
                }
                mma16816<SPLIT>(sc[j], a[0][ks], b[0][2 * kk], b[0][2 * kk + 1]);
            }
        }
    }
}

template <bool SPLIT, int D>
__device__ __forceinline__ void load_a(uint32_t (&a)[SPLIT ? 2 : 1][D / 16][4], const uint16_t *sq, int m0, int lane)
{
    constexpr int NP = SPLIT ? 2 : 1, kPitch = GaShape<D>::kPitch;
#pragma unroll
    for (int pl = 0; pl < NP; ++pl)
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks) ldsm_x4(a[pl][ks], sq + (pl * kTile + m0 + (lane & 15)) * kPitch + ks * 16 + (lane >> 4) * 8);
}

template <bool SPLIT, int D>
__global__ void __launch_bounds__(kTcThreads) gen_attention_mma_kernel(const __grid_constant__ GaParams P)
{
    constexpr int NP = SPLIT ? 2 : 1, kPitch = GaShape<D>::kPitch;
    extern __shared__ uint4 s_ga[];
    uint16_t *sq = reinterpret_cast<uint16_t *>(s_ga), *sk = sq + NP * kTile * kPitch, *sv = sk + NP * kTile * kPitch;
    int *s_ky = reinterpret_cast<int *>(sv + NP * kTile * kPitch), *s_kx = s_ky + kTile;
    float *s_tx = reinterpret_cast<float *>(s_kx + kTile), *s_ty = s_tx + kTile * (P.Wk + 1);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3, m0 = warp * 16;
    const int head = blockIdx.y, n = blockIdx.z;
    const int hw = P.H * P.W, q0 = blockIdx.x * kTile, nq = min(kTile, hw - q0), nk = P.Hk * P.Wk;
    const long long qtok = (long long)n * hw + q0, ktok = (long long)n * nk;
    const int col0 = head * D;
    const int rows[2] = {m0 + g, m0 + g + 8};

    // ---- position rows: Tx[q][kx] = Qp[q] . Px[qx - s kx], Ty[q][ky] = Qp[q] . Py[qy - s ky]
    if (P.qp) {
        stage_rows<NP, D>(sq, static_cast<const uint16_t *>(P.qp), qtok, nq, P.ldq, col0);
        cp_wait_all();
        __syncthreads();
        uint32_t ap[NP][D / 16][4];
        load_a<SPLIT, D>(ap, sq, m0, lane);
#pragma unroll 1
        for (int axis = 0; axis < 2; ++axis) {
            const int extent = axis ? P.H : P.W, kext = axis ? P.Hk : P.Wk;
            const int R = extent + P.s * (kext - 1);
            const uint16_t *tab = static_cast<const uint16_t *>(axis ? P.py : P.px);
            float *dst = axis ? s_ty : s_tx;
            int qc[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int qi = q0 + min(rows[h], nq - 1);
                qc[h] = (axis ? qi / P.W : qi % P.W) + P.s * (kext - 1);     // table row of the offset to key coordinate 0
            }
#pragma unroll 1
            for (int r0 = 0; r0 < R; r0 += kTile) {
                __syncthreads();                                              // the previous step's readers of sk are done
                stage_rows<NP, D>(sk, tab, r0, min(kTile, R - r0), P.C, col0);
                cp_wait_all();
                __syncthreads();
                float sc[8][4];
                mma_rows<SPLIT, D>(sc, ap, sk, lane);
#pragma unroll
                for (int j = 0; j < 8; ++j)
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int h = e >> 1, r = r0 + 8 * j + 2 * t4 + (e & 1);
                        const int diff = qc[h] - r;                           // = s * kx for the key column this row serves
                        if (r < R && diff >= 0 && (diff & (P.s - 1)) == 0 && (diff >> (P.s - 1)) < kext)
                            dst[rows[h] * (kext + 1) + (diff >> (P.s - 1))] = sc[j][e];
                    }
            }
        }
    }
    // ---- content queries
    uint32_t aq[NP][D / 16][4];
    __syncthreads();
    if (P.qc) {
        stage_rows<NP, D>(sq, static_cast<const uint16_t *>(P.qc), qtok, nq, P.ldq, col0);
        cp_wait_all();
        __syncthreads();
        load_a<SPLIT, D>(aq, sq, m0, lane);
    }
    // ---- stream the keys: online softmax over tiles of kTile keys
    float o[D / 8][4];
#pragma unroll
    for (int jn = 0; jn < D / 8; ++jn) o[jn][0] = o[jn][1] = o[jn][2] = o[jn][3] = 0.f;
    float mx[2] = {-3.0e38f, -3.0e38f}, den[2] = {0.f, 0.f};
#pragma unroll 1
    for (int k0 = 0; k0 < nk; k0 += kTile) {
        const int nkt = min(kTile, nk - k0);
        __syncthreads();                                                      // the previous tile's readers are done
        if (P.k) stage_rows<NP, D>(sk, static_cast<const uint16_t *>(P.k), ktok + k0, nkt, P.ldkv, col0);
        stage_rows<NP, D>(sv, static_cast<const uint16_t *>(P.v), ktok + k0, nkt, P.ldkv, col0);
        if (tid < kTile) {
            const int kj = k0 + tid, ky = kj / P.Wk;
            s_ky[tid] = tid < nkt ? ky : -1;
            s_kx[tid] = kj - ky * P.Wk;
        }
        cp_wait_all();
        __syncthreads();
        float sc[8][4];
        if (P.qc) {
            mma_rows<SPLIT, D>(sc, aq, sk, lane);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) sc[j][0] = sc[j][1] = sc[j][2] = sc[j][3] = 0.f;
        }
        float tmax[2] = {-3.0e38f, -3.0e38f};
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int h = e >> 1, c = 8 * j + 2 * t4 + (e & 1);
                const int ky = s_ky[c];
                float v = -3.0e38f;
                if (ky >= 0) {
                    v = sc[j][e];
                    if (P.qp) v += s_tx[rows[h] * (P.Wk + 1) + s_kx[c]] + s_ty[rows[h] * (P.Hk + 1) + ky];
                    tmax[h] = fmaxf(tmax[h], v);
                }
                sc[j][e] = v;
            }
        float corr[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            tmax[h] = fmaxf(tmax[h], __shfl_xor_sync(0xffffffffu, tmax[h], 1));
            tmax[h] = fmaxf(tmax[h], __shfl_xor_sync(0xffffffffu, tmax[h], 2));
            const float mn = fmaxf(mx[h], tmax[h]);                           // finite: every tile holds a key
            corr[h] = expf(mx[h] - mn);
            mx[h] = mn;
            den[h] *= corr[h];
        }
#pragma unroll
        for (int jn = 0; jn < D / 8; ++jn) { o[jn][0] *= corr[0]; o[jn][1] *= corr[0]; o[jn][2] *= corr[1]; o[jn][3] *= corr[1]; }
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float p = expf(sc[j][e] - mx[e >> 1]);                  // a missing key: exp(-3e38 - m) = 0
                sc[j][e] = p;
                den[e >> 1] += p;
            }
        // O += P V: the accumulator fragments of two neighbouring 8-key tiles are the A fragment of one 16-key step
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            uint32_t ph[4], pl_[4];
            split_pair<SPLIT>(sc[2 * kk][0], sc[2 * kk][1], ph[0], pl_[0]);
            split_pair<SPLIT>(sc[2 * kk][2], sc[2 * kk][3], ph[1], pl_[1]);
            split_pair<SPLIT>(sc[2 * kk + 1][0], sc[2 * kk + 1][1], ph[2], pl_[2]);
            split_pair<SPLIT>(sc[2 * kk + 1][2], sc[2 * kk + 1][3], ph[3], pl_[3]);
#pragma unroll
            for (int np = 0; np < D / 16; ++np) {
                uint32_t bv[NP][4];
#pragma unroll
                for (int pl = 0; pl < NP; ++pl)
                    ldsm_x4_trans(bv[pl], sv + (pl * kTile + 16 * kk + ((lane >> 3) & 1) * 8 + (lane & 7)) * kPitch + 16 * np + (lane >> 4) * 8);
                mma16816<SPLIT>(o[2 * np], pl_, bv[0][0], bv[0][1]); mma16816<SPLIT>(o[2 * np + 1], pl_, bv[0][2], bv[0][3]);    // p_lo v_hi
                if (SPLIT) { mma16816<SPLIT>(o[2 * np], ph, bv[NP - 1][0], bv[NP - 1][1]); mma16816<SPLIT>(o[2 * np + 1], ph, bv[NP - 1][2], bv[NP - 1][3]); }
                mma16816<SPLIT>(o[2 * np], ph, bv[0][0], bv[0][1]); mma16816<SPLIT>(o[2 * np + 1], ph, bv[0][2], bv[0][3]);
            }
        }
    }
    // ---- normalise and store: the output is a convex combination of V rows, so it stays within their (fp16) range
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        den[h] += __shfl_xor_sync(0xffffffffu, den[h], 1);
        den[h] += __shfl_xor_sync(0xffffffffu, den[h], 2);
        if (rows[h] >= nq) continue;
        const float inv = 1.0f / den[h];
        uint16_t *dst = static_cast<uint16_t *>(P.out) + (qtok + rows[h]) * NP * (long long)P.C + col0 + 2 * t4;
#pragma unroll
        for (int jn = 0; jn < D / 8; ++jn) {
            float x = o[jn][2 * h] * inv, y = o[jn][2 * h + 1] * inv;
            if (SPLIT) { x = fminf(fmaxf(x, -65504.f), 65504.f); y = fminf(fmaxf(y, -65504.f), 65504.f); }
            uint32_t hi, lo;
            split_pair<SPLIT>(x, y, hi, lo);
            *reinterpret_cast<uint32_t *>(dst + 8 * jn) = hi;
            if (SPLIT) *reinterpret_cast<uint32_t *>(dst + P.C + 8 * jn) = lo;
        }
    }
}

// fp32 on the CUDA cores: thread = query; per key the logit Qc . K (channel order) + Tx + Ty, then the online softmax update
template <int D>
__global__ void __launch_bounds__(kF32Threads) gen_attention_f32_kernel(const __grid_constant__ GaParams P)
{
    extern __shared__ float4 s_ga32[];
    float *sk = reinterpret_cast<float *>(s_ga32), *sv = sk + kTile * D;
    int *s_ky = reinterpret_cast<int *>(sv + kTile * D), *s_kx = s_ky + kTile;
    float *s_tx = reinterpret_cast<float *>(s_kx + kTile), *s_ty = s_tx + kTile * (P.Wk + 1);
    const int tid = threadIdx.x, head = blockIdx.y, n = blockIdx.z;
    const int hw = P.H * P.W, q0 = blockIdx.x * kTile, nk = P.Hk * P.Wk;
    const int qi = min(q0 + tid, hw - 1);                                     // rows past the map compute on a clamped query
    const long long qtok = (long long)n * hw + qi, ktok = (long long)n * nk;
    const int col0 = head * D;
    const int qy = qi / P.W, qx = qi - qy * P.W;
    if (P.qp) {
        float qp[D];
        const float *src = static_cast<const float *>(P.qp) + qtok * P.ldq + col0;
#pragma unroll
        for (int c = 0; c < D; c += 4) { const float4 t = *reinterpret_cast<const float4 *>(src + c); qp[c] = t.x; qp[c + 1] = t.y; qp[c + 2] = t.z; qp[c + 3] = t.w; }
#pragma unroll 1
        for (int axis = 0; axis < 2; ++axis) {
            const int kext = axis ? P.Hk : P.Wk, base = (axis ? qy : qx) + P.s * (kext - 1);
            const float *tab = static_cast<const float *>(axis ? P.py : P.px) + col0;
            float *dst = (axis ? s_ty : s_tx) + tid * (kext + 1);
#pragma unroll 1
            for (int kc = 0; kc < kext; ++kc) {
                const float *row = tab + (long long)(base - P.s * kc) * P.C;
                float acc = 0.f;
#pragma unroll
                for (int c = 0; c < D; c += 4) {
                    const float4 t = *reinterpret_cast<const float4 *>(row + c);
                    acc = fmaf(qp[c], t.x, acc); acc = fmaf(qp[c + 1], t.y, acc); acc = fmaf(qp[c + 2], t.z, acc); acc = fmaf(qp[c + 3], t.w, acc);
                }
                dst[kc] = acc;
            }
        }
    }
    float qc[D], o[D];
    if (P.qc) {
        const float *src = static_cast<const float *>(P.qc) + qtok * P.ldq + col0;
#pragma unroll
        for (int c = 0; c < D; c += 4) { const float4 t = *reinterpret_cast<const float4 *>(src + c); qc[c] = t.x; qc[c + 1] = t.y; qc[c + 2] = t.z; qc[c + 3] = t.w; }
    }
#pragma unroll
    for (int c = 0; c < D; ++c) o[c] = 0.f;
    float mx = -3.0e38f, den = 0.f;
#pragma unroll 1
    for (int k0 = 0; k0 < nk; k0 += kTile) {
        const int nkt = min(kTile, nk - k0);
        __syncthreads();
        for (int i = tid; i < nkt * (D / 4); i += kF32Threads) {
            const int row = i / (D / 4), c = (i % (D / 4)) * 4;
            const long long off = (ktok + k0 + row) * P.ldkv + col0 + c;
            if (P.k) *reinterpret_cast<float4 *>(sk + row * D + c) = *reinterpret_cast<const float4 *>(static_cast<const float *>(P.k) + off);
            *reinterpret_cast<float4 *>(sv + row * D + c) = *reinterpret_cast<const float4 *>(static_cast<const float *>(P.v) + off);
        }
        {
            const int kj = k0 + tid, ky = kj / P.Wk;
            s_ky[tid] = ky;
            s_kx[tid] = kj - ky * P.Wk;
        }
        __syncthreads();
#pragma unroll 1
        for (int j = 0; j < nkt; ++j) {
            float e = 0.f;
            if (P.qc) {
                const float *kr = sk + j * D;
#pragma unroll
                for (int c = 0; c < D; ++c) e = fmaf(qc[c], kr[c], e);
            }
            if (P.qp) e += s_tx[tid * (P.Wk + 1) + s_kx[j]] + s_ty[tid * (P.Hk + 1) + s_ky[j]];
            if (e > mx) {
                const float corr = expf(mx - e);
                den *= corr;
#pragma unroll
                for (int c = 0; c < D; ++c) o[c] *= corr;
                mx = e;
            }
            const float p = expf(e - mx);
            den += p;
            const float *vr = sv + j * D;
#pragma unroll
            for (int c = 0; c < D; ++c) o[c] = fmaf(p, vr[c], o[c]);
        }
    }
    if (q0 + tid >= hw) return;
    const float inv = 1.0f / den;
    float *dst = static_cast<float *>(P.out) + qtok * P.C + col0;
#pragma unroll
    for (int c = 0; c < D; c += 4) *reinterpret_cast<float4 *>(dst + c) = make_float4(o[c] * inv, o[c + 1] * inv, o[c + 2] * inv, o[c + 3] * inv);
}

inline bool al16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// format: 0 bf16, 1 f16x3, 2 fp32
int plan(const orp_gen_attention_args *a, int format, orp_gen_attention_plan *out, GaParams *prm)
{
    if (!a || !out || format < 0 || format > 2) return fail(ORP_EINVAL, "gen_attention_plan: needs arguments, a plan and format 0, 1 or 2");
    if (a->N < 1 || a->H < 1 || a->W < 1 || a->Hk < 1 || a->Wk < 1 || a->N > 65535 || a->heads < 1 || a->heads > 65535)
        return fail(ORP_EINVAL, "gen_attention: needs N, H, W, Hk, Wk >= 1, N <= 65535 and 1 <= heads <= 65535");
    if (a->C % a->heads || (a->C / a->heads != 32 && a->C / a->heads != 64))
        return fail(ORP_EINVAL, "gen_attention: runs head dimensions C / heads of 32 and 64");
    if (a->kv_stride != 1 && a->kv_stride != 2) return fail(ORP_EINVAL, "gen_attention: kv_stride must be 1 or 2");
    if (a->ld_q % 8 || a->ld_kv % 8 || a->ld_q < a->C || a->ld_kv < a->C)
        return fail(ORP_EINVAL, "gen_attention: ld_q and ld_kv must be multiples of 8 and at least C");
    if (!a->out || !a->v) return fail(ORP_EINVAL, "gen_attention: out and v must not be NULL");
    if (!a->q_c != !a->k) return fail(ORP_EINVAL, "gen_attention: q_c and k are given together or not at all");
    if (!a->q_p != !a->pos_x || !a->q_p != !a->pos_y)
        return fail(ORP_EINVAL, "gen_attention: q_p, pos_x and pos_y are given together or not at all");
    const void *ptrs[7] = {a->q_c, a->q_p, a->k, a->v, a->pos_x, a->pos_y, a->out};
    for (const void *p : ptrs)
        if (!al16(p)) return fail(ORP_EINVAL, "gen_attention: every pointer must be 16-byte aligned");
    for (int i = 0; i < 6; ++i)
        if (ptrs[i] && ptrs[i] == a->out) return fail(ORP_EINVAL, "gen_attention: out must be distinct from every input");
    if (a->q_p && (a->Hk != (a->H + a->kv_stride - 1) / a->kv_stride || a->Wk != (a->W + a->kv_stride - 1) / a->kv_stride))
        return fail(ORP_EINVAL, "gen_attention: with a position term Hk and Wk must be ceil(H / kv_stride) and ceil(W / kv_stride)");
    const int d = a->C / a->heads;
    GaParams p{a->q_c, a->q_p, a->k, a->v, a->pos_x, a->pos_y, a->out, a->N, a->H, a->W, a->Hk, a->Wk, a->kv_stride, a->C, a->heads,
               a->ld_q, a->ld_kv};
    const long long tiles = ((long long)a->H * a->W + kTile - 1) / kTile;
    const long long smem = (format == 2 ? (d == 32 ? GaShape<32>::f32_tiles_bytes() : GaShape<64>::f32_tiles_bytes())
                                        : (d == 32 ? GaShape<32>::tc_tiles_bytes(format == 1) : GaShape<64>::tc_tiles_bytes(format == 1)))
                           + 2 * kTile * 4 + tables_bytes(p);
    if (tiles > 0x7fffffff) return fail(ORP_EINVAL, "gen_attention: H * W too large");
    if (smem > kMaxSmem)
        return fail(ORP_EINVAL, "gen_attention: the per-query position rows (Hk + Wk + 2 floats each) exceed the shared memory of a CTA");
    *out = orp_gen_attention_plan{};
    out->head_dim = d;
    out->queries_per_cta = kTile;
    out->threads = format == 2 ? kF32Threads : kTcThreads;
    out->grid_x = (int)tiles;
    out->grid_y = a->heads;
    out->grid_z = a->N;
    out->smem_bytes = (int)smem;
    out->rx = a->q_p ? a->W + a->kv_stride * (a->Wk - 1) : 0;
    out->ry = a->q_p ? a->H + a->kv_stride * (a->Hk - 1) : 0;
    out->content = a->q_c != nullptr;
    out->position = a->q_p != nullptr;
    if (prm) *prm = p;
    return ORP_OK;
}

template <auto Kern>
int launch(const orp_gen_attention_plan &pl, const GaParams &p, void *stream)
{
    static int opted[64];                        // opt this kernel in to the full dynamic shared memory, once per device
    int dev = 0;
    ORP_CUDA(cudaGetDevice(&dev));
    if (dev >= 64 || !__atomic_load_n(&opted[dev], __ATOMIC_ACQUIRE)) {
        ORP_CUDA(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
        if (dev < 64) __atomic_store_n(&opted[dev], 1, __ATOMIC_RELEASE);
    }
    Kern<<<dim3(pl.grid_x, pl.grid_y, pl.grid_z), pl.threads, pl.smem_bytes, static_cast<cudaStream_t>(stream)>>>(p);
    ORP_LAUNCHED();
    return ORP_OK;
}

int run(const orp_gen_attention_args *a, int format, void *stream)
{
    orp_gen_attention_plan pl;
    GaParams p;
    int rc = plan(a, format, &pl, &p);
    if (rc || (rc = ensure_device())) return rc;
    if (format == 2)
        return pl.head_dim == 32 ? launch<gen_attention_f32_kernel<32>>(pl, p, stream) : launch<gen_attention_f32_kernel<64>>(pl, p, stream);
    if (format == 1)
        return pl.head_dim == 32 ? launch<gen_attention_mma_kernel<true, 32>>(pl, p, stream) : launch<gen_attention_mma_kernel<true, 64>>(pl, p, stream);
    return pl.head_dim == 32 ? launch<gen_attention_mma_kernel<false, 32>>(pl, p, stream) : launch<gen_attention_mma_kernel<false, 64>>(pl, p, stream);
}

// y = x + row[n]: one item = (pixel, 8 channels)
template <class A>
__global__ void __launch_bounds__(256) bcast_add_kernel(const typename A::T *x, int N, int HW, int C, const float *row, typename A::T *y,
                                                        unsigned int *ovf)
{
    const int c8 = C / 8;
    const size_t total = (size_t)N * HW * c8;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % c8) * 8;
        const size_t pix = i / c8, n = pix / HW;
        float v[8], r[8];
        A::ld8(x, (long long)pix, C, c, v);
        ActF32::ld8(row, (long long)n, C, c, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] += r[j];
        store8<A>(y, (long long)pix, C, c, v, ovf);
    }
}

template <class A>
int bcast_add(const void *x, int N, int H, int W, int C, const float *row, void *y, void *stream, const char *name)
{
    if (!x || !row || !y || bad_dims(N, H, W, C) || !aligned16(x) || !aligned16(row) || !aligned16(y) || x == y)
        return fail(ORP_EINVAL, "%s: needs distinct 16-byte aligned x, row and y, N, H, W >= 1 and C a multiple of 8", name);
    unsigned int *ovf;
    int rc = overflow_ptr(A::planes == 2, ovf, name);
    if (rc || (rc = ensure_device())) return rc;
    bcast_add_kernel<A><<<grid_for((size_t)N * H * W * (C / 8), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const typename A::T *>(x), N, H * W, C, row, static_cast<typename A::T *>(y), ovf);
    ORP_LAUNCHED();
    return ORP_OK;
}

}  // namespace
}  // namespace orp

using namespace orp;

/* see include/orp_b200_attention.h */
extern "C" int orp_gen_attention_bf16(const orp_gen_attention_args *a, void *stream) { return run(a, 0, stream); }
extern "C" int orp_gen_attention_f16x3(const orp_gen_attention_args *a, void *stream) { return run(a, 1, stream); }
extern "C" int orp_gen_attention_f32(const orp_gen_attention_args *a, void *stream) { return run(a, 2, stream); }

extern "C" int orp_gen_attention_make_plan(const orp_gen_attention_args *a, int format, orp_gen_attention_plan *out)
{
    return plan(a, format, out, nullptr);
}

extern "C" int orp_gen_attention_bcast_add_bf16(const void *x, int N, int H, int W, int C, const float *row, void *y, void *stream)
{
    return bcast_add<Act<false>>(x, N, H, W, C, row, y, stream, "gen_attention_bcast_add_bf16");
}
extern "C" int orp_gen_attention_bcast_add_f16x3(const void *x, int N, int H, int W, int C, const float *row, void *y, void *stream)
{
    return bcast_add<Act<true>>(x, N, H, W, C, row, y, stream, "gen_attention_bcast_add_f16x3");
}
extern "C" int orp_gen_attention_bcast_add_f32(const float *x, int N, int H, int W, int C, const float *row, float *y, void *stream)
{
    return bcast_add<ActF32>(x, N, H, W, C, row, y, stream, "gen_attention_bcast_add_f32");
}
