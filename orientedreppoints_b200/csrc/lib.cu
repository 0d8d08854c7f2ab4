// lib.cu - process-wide state of liborp_b200.so: error string, launch counter, device gate.
#include "common.cuh"

namespace orp {

thread_local char g_err[512] = "";
int64_t g_launches = 0;
int g_timing = 0;

int ensure_device()
{
    static thread_local int checked_dev = -1;
    int dev = 0;
    ORP_CUDA(cudaGetDevice(&dev));
    if (dev == checked_dev) return ORP_OK;
    cudaDeviceProp prop;
    ORP_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9) {
        snprintf(g_err, sizeof(g_err),
                 "liborp_b200 is built for sm_90a (H100) only; device %d is sm_%d%d (no fallback path exists)", dev,
                 prop.major, prop.minor);
        return ORP_ENOGPU;
    }
    // keep freed scratch cached in the stream-ordered pool
    cudaMemPool_t pool;
    ORP_CUDA(cudaDeviceGetDefaultMemPool(&pool, dev));
    uint64_t thresh = ~0ull;
    ORP_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
    checked_dev = dev;
    return ORP_OK;
}

int device_sms(int &sms)
{
    static thread_local int dev_known = -1, sms_known = 0;
    int dev = 0;
    ORP_CUDA(cudaGetDevice(&dev));
    if (dev != dev_known) {
        ORP_CUDA(cudaDeviceGetAttribute(&sms_known, cudaDevAttrMultiProcessorCount, dev));
        dev_known = dev;
    }
    sms = sms_known;
    return ORP_OK;
}

}  // namespace orp

extern "C" const char *orp_last_error(void) { return orp::g_err; }
extern "C" void orp_set_timing(int on) { orp::g_timing = on; }
extern "C" int orp_version(void) { return 100; }
extern "C" int orp_compiled_sm(void) { return 90; }
extern "C" int64_t orp_launch_count(void) { return __atomic_load_n(&orp::g_launches, __ATOMIC_RELAXED); }
extern "C" void orp_reset_launch_count(void) { __atomic_store_n(&orp::g_launches, 0, __ATOMIC_RELAXED); }
