// Library-level entry points: error string, version, device probe.
#include "common.cuh"
#include "../../include/fastmot_b200.h"
#include <string.h>

static thread_local char g_last_error[512] = "";

extern "C" void fm_set_last_error(const char* msg) {
    strncpy(g_last_error, msg ? msg : "", sizeof g_last_error - 1);
    g_last_error[sizeof g_last_error - 1] = 0;
}

extern "C" const char* fm_last_error(void) { return g_last_error; }

extern "C" int fm_version(void) { return 103; }

extern "C" int fm_device_ok(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        fm_set_last_error("no CUDA device");
        return 0;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 0;
    if (p.major != 9) {
        fm_set_last_error("device is not sm_90 (Hopper H100)");
        return 0;
    }
    return 1;
}

extern "C" int fm_memcpy_async(void* dst, const void* src, long long bytes, void* stream) {
    if (bytes <= 0) return FM_OK;
    cudaError_t e = cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDefault, (cudaStream_t)stream);
    if (e != cudaSuccess) {
        fm_set_last_error(cudaGetErrorString(e));
        return FM_ERR_CUDA;
    }
    return FM_OK;
}

extern "C" int fm_host_is_pinned(const void* p) {
    cudaPointerAttributes a;
    cudaError_t e = cudaPointerGetAttributes(&a, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return a.type == cudaMemoryTypeHost ? 1 : 0;
}

// Kernel-launch accounting for bench.py's `gpu_launches` (one increment per C-ABI launch site; multi-kernel entry
// points add their extra kernels explicitly).
static long long g_launches = 0;
extern "C" void fm_count_launches(int n) { __atomic_fetch_add(&g_launches, (long long)n, __ATOMIC_RELAXED); }
extern "C" long long fm_launch_count(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }
