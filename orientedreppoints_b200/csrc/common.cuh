// common.cuh - error plumbing, launch accounting and stream-ordered scratch memory shared by
// every translation unit of liborp_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/orp_b200.h"

namespace orp {

extern thread_local char g_err[512];
extern int64_t g_launches;
extern int g_timing;                     // orp_set_timing(): bracket dominant kernels with CUDA events

inline int fail(int code, const char *fmt, const char *a = "", const char *b = "")
{
    snprintf(g_err, sizeof(g_err), fmt, a, b);
    return code;
}

#define ORP_CUDA(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) return ::orp::fail(ORP_ECUDA, "%s: %s", #expr, cudaGetErrorString(e__)); \
    } while (0)

#define ORP_LAUNCHED()                                                                          \
    do {                                                                                        \
        __atomic_add_fetch(&::orp::g_launches, 1, __ATOMIC_RELAXED);                            \
        cudaError_t e__ = cudaGetLastError();                                                   \
        if (e__ != cudaSuccess) return ::orp::fail(ORP_ECUDA, "kernel launch: %s", cudaGetErrorString(e__)); \
    } while (0)

inline void count_launches(int n) { __atomic_add_fetch(&g_launches, n, __ATOMIC_RELAXED); }

// one-time per-device setup: refuse anything that is not compute capability 9.x, and keep
// freed scratch in the stream-ordered pool so repeated calls do not hit the driver allocator.
int ensure_device();

// RAII scratch arena on a stream (cudaMallocAsync / cudaFreeAsync).
struct Scratch {
    cudaStream_t st;
    void *ptrs[48];
    int n = 0;
    explicit Scratch(cudaStream_t s) : st(s) {}
    ~Scratch() { for (int i = 0; i < n; ++i) cudaFreeAsync(ptrs[i], st); }
    template <typename T> T *get(size_t count)
    {
        void *p = nullptr;
        size_t bytes = (count ? count : 1) * sizeof(T);
        if (n >= 48 || cudaMallocAsync(&p, bytes, st) != cudaSuccess) return nullptr;
        ptrs[n++] = p;
        return static_cast<T *>(p);
    }
};

// nms.cu: device-resident greedy rotated NMS (see orp_rnms); flags_out = uint8 survivor flags by original index
int run_nms(const float *dets, const int32_t *segments, int n, double thr, int iou_mode, int union_mode,
            int order, int64_t *keep_out, int32_t *num_out, cudaStream_t st, uint8_t *flags_out, bool no_sync,
            int seg_limit /* exclusive bound on segment ids, 0 = unknown */,
            int32_t *overflow_out /* optional device int: set to 1 when the candidate list overflowed (no_sync callers) */);

static inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

// key bits that hold every value in [0, v]
inline int key_bits(uint64_t v)
{
    int b = 1;
    while (b < 64 && (v >> b)) ++b;
    return b;
}

// sort key of a float: ascending key order == ascending float order
__device__ __forceinline__ uint32_t orderable(float f)
{
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// multiprocessors of the current device, looked up once per device
int device_sms(int &sms);

// streaming multiprocessors of an H100 SXM: caps of grid-stride launches are multiples of it
constexpr int kNumSMs = 132;

// blocks of a grid-stride launch over `items`: enough for one item per thread, at most 16 per SM, at least one
inline int grid_for(size_t items, int threads)
{
    const size_t g = (items + threads - 1) / threads;
    const size_t cap = kNumSMs * 16;
    return (int)(g < cap ? (g ? g : 1) : cap);
}

}  // namespace orp
